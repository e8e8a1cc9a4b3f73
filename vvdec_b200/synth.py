"""Synthetic post-parse content (SURVEY.md §8d): there is no VVC bitstream or encoder on the box, so the
work lists a flattener would emit from VVdeC's parsed Picture are drawn from a seeded generator instead.
Everything here is host-side input preparation (numpy); no pixel arithmetic of the hot path lives here."""
import ctypes as C
import numpy as np
from . import abi


def partition(rng, W, H, ctu=128, min_dim=4, min_area=32, p_split=None):
    """Random QT+BT partition of a WxH picture into CUs. Returns int array [n,4] = x,y,w,h (luma).
    Blocks crossing the picture boundary are split until they fit (implicit boundary splits)."""
    out = []
    p_split = p_split or {128: 0.94, 64: 0.68, 32: 0.6, 16: 0.6, 8: 0.5, 4: 0.0}

    def rec(x, y, w, h):
        if x >= W or y >= H:
            return
        cross_x, cross_y = x + w > W, y + h > H
        big = max(w, h)
        if cross_x or cross_y:
            if cross_x and cross_y or (w == h and w > 64):
                mode = "q"
            else:
                mode = "v" if cross_x else "h"
        else:
            r = rng.random()
            if r >= p_split.get(big, 0.0):
                out.append((x, y, w, h)); return
            opts = []
            if w == h and w >= 16: opts += ["q", "q"]
            if w >= 2 * min_dim and (w // 2) * h >= min_area and w <= 64: opts.append("v")
            if h >= 2 * min_dim and w * (h // 2) >= min_area and h <= 64: opts.append("h")
            if not opts:
                out.append((x, y, w, h)); return
            mode = opts[rng.integers(0, len(opts))]
        if mode == "q":
            hw, hh = w // 2, h // 2
            for dy in (0, hh):
                for dx in (0, hw):
                    rec(x + dx, y + dy, hw, hh)
        elif mode == "v":
            rec(x, y, w // 2, h); rec(x + w // 2, y, w // 2, h)
        else:
            rec(x, y, w, h // 2); rec(x, y + h // 2, w, h // 2)

    for cy in range(0, H, ctu):
        for cx in range(0, W, ctu):
            rec(cx, cy, ctu, ctu)
    return np.array(out, np.int32).reshape(-1, 4)


def _laplace_levels(rng, n, heavy=False):
    v = rng.laplace(0, 2.0 if not heavy else 400.0, size=n)
    return np.clip(np.rint(v), -32768, 32767).astype(np.int16)


TU_INV_SCALES = ((40, 45, 51, 57, 64, 72), (57, 64, 72, 80, 90, 102))      # g_invQuantScales: [sqrt2 shape][QP % 6]


def tu_dequant(qp, bit_depth, l2w, l2h, ts=False, dep_quant=False, scaling=False):
    """(rightShift, inBits, scale) of a TU record, as the flattener derives them (vvdec_glue/flatten_tu.h): qp = QP' (QP + 6 (bitDepth - 8)),
    at least 4 under transform skip; dependent quantisation adds 1 to QP and to the shift, explicit scaling lists add 4 to the shift."""
    sqrt2 = (not ts) and ((l2w + l2h) & 1)
    q = max(qp, 4) if ts else qp
    per, rem = ((q + 1) // 6, (q + 1) % 6) if dep_quant else (q // 6, q % 6)
    tr_shift = 15 - bit_depth - ((l2w + l2h) >> 1) + (-1 if sqrt2 else 0)
    right_shift = 6 + (1 if dep_quant else 0) - ((0 if ts else tr_shift) + per) + (4 if scaling else 0)
    return right_shift, min(16, 32 + right_shift - 7), TU_INV_SCALES[1 if sqrt2 else 0][rem]


def gen_tus(rng, cus, bit_depth=10, p_cbf=0.5, p_mts=0.2, p_lfnst=0.1, p_ts=0.05, p_bdpcm=0.03, p_jccr=0.1,
            p_full=0.3, chroma=True, heavy=0.02, dep_quant=True, p_intra=0.15, scaling=None):
    """TU records + packed level arena for a CU list (one TU per <=64x64 tile of each CU, all 3 components).
    Mirrors what the flattener (vvdec_glue/flatten_tu.h) derives from parsed TUs; QP drawn uniformly in 22..37.
    scaling: None, or the dict of gen_scaling_lists(): non-TS, non-LFNST TUs then use explicit scaling lists (Quant.cpp:309-312):
    B200_TU_SCALING, slOff -> the table of their (log2w, log2h), right shift + 4."""
    recs, coefs = [], []
    ncoef = 0
    for (cx, cy, cw, ch) in cus:
        if rng.random() >= p_cbf:
            continue
        qp = int(rng.integers(22, 38)) + 6 * (bit_depth - 8)
        intra = rng.random() < p_intra
        for ty in range(cy, cy + ch, 64):
            for tx in range(cx, cx + cw, 64):
                tw, th = min(64, cw), min(64, ch)
                jccr = chroma and rng.random() < p_jccr
                for comp in ((0, 1, 2) if chroma else (0,)):
                    w, h = (tw, th) if comp == 0 else (tw >> 1, th >> 1)
                    x, y = (tx, ty) if comp == 0 else (tx >> 1, ty >> 1)
                    if min(w, h) < 2 or (comp and rng.random() < 0.3 and not jccr):
                        continue
                    ict = 0
                    if comp and jccr:
                        if comp == 2: continue
                        ict = int(rng.choice([-3, -2, -1, 1, 2, 3]))
                        if abs(ict) == 3: comp = 2
                    l2w, l2h = int(np.log2(w)), int(np.log2(h))
                    flags, tr, lfnst = 0, 0, 0
                    r = rng.random()
                    maxX = maxY = None
                    if w <= 32 and h <= 32 and r < p_bdpcm and intra:
                        flags = abi.TU_TS | (abi.TU_BDPCM_H if rng.random() < 0.5 else abi.TU_BDPCM_V)
                        maxX, maxY = w - 1, h - 1
                    elif w <= 32 and h <= 32 and r < p_bdpcm + p_ts:
                        flags = abi.TU_TS
                    elif comp == 0 and min(w, h) >= 4 and max(w, h) <= 32 and r < p_bdpcm + p_ts + p_mts:
                        th_, tv_ = rng.choice([abi.TR_DST7, abi.TR_DCT8], size=2)
                        tr = int(th_) | (int(tv_) << 2)
                    elif intra and min(w, h) >= 4 and r < p_bdpcm + p_ts + p_mts + p_lfnst:
                        lf_set = int(rng.integers(0, 4))
                        lfnst = int(rng.integers(1, 3)) | (lf_set << 2) | ((int(rng.integers(0, 2)) if lf_set else 0) << 4)
                    if maxX is None:
                        limx = min(w, 32) if not (tr & 3 and w == 32) else 16
                        limy = min(h, 32) if not ((tr >> 2) & 3 and h == 32) else 16
                        if lfnst:
                            # at most 16 (8 for 4x4/8x8) levels in scan order, all inside the first 4x4 coefficient group
                            maxX, maxY = 3, 3
                        elif rng.random() < p_full:
                            maxX, maxY = limx - 1, limy - 1
                        else:
                            maxX = min(limx - 1, int(rng.geometric(0.25)) - 1)
                            maxY = min(limy - 1, int(rng.geometric(0.25)) - 1)
                        if not (flags & abi.TU_TS) and not (maxX == 0 and maxY == 0):
                            # the parser reports the coded corner in whole coefficient groups (CABACReader.cpp:2447-2452): 4x4, or
                            # 2x8 / 8x2 for 2-wide / 2-high blocks; only a lone DC coefficient gives (0,0)
                            cgw, cgh = (2, 8) if w == 2 else (8, 2) if h == 2 else (4, 4)
                            maxX = min(limx, (maxX // cgw + 1) * cgw) - 1
                            maxY = min(limy, (maxY // cgh + 1) * cgh) - 1
                    is_ts = bool(flags & abi.TU_TS)
                    sl_off = 0
                    use_sl = scaling is not None and not is_ts and not lfnst
                    if use_sl:
                        flags |= abi.TU_SCALING; sl_off = scaling["off"][(l2w, l2h)]
                    right_shift, in_bits, scale = tu_dequant(qp, bit_depth, l2w, l2h, is_ts, dep_quant and not is_ts, use_sl)
                    n = (maxX + 1) * (maxY + 1)
                    lv = _laplace_levels(rng, n, rng.random() < heavy)
                    if lfnst:
                        # zero everything outside the first 8 scan positions (x+y<=2 covers 6 of them: safe subset)
                        yy, xx = np.divmod(np.arange(n), maxX + 1)
                        lv[(xx + yy) > 2] = 0
                    if lv[-1] == 0: lv[-1] = 1
                    recs.append((x, y, l2w, l2h, comp, flags, maxX, maxY, tr, lfnst, ict, right_shift, in_bits, scale, ncoef, sl_off, (0, 0)))
                    coefs.append(lv); ncoef += n
    tus = np.array(recs, dtype=abi.TU_DTYPE) if recs else np.zeros(0, abi.TU_DTYPE)
    arena = np.concatenate(coefs) if coefs else np.zeros(0, np.int16)
    return tus, arena


def gen_scaling_lists(rng):
    """One dequantisation table per block shape, laid out as Quant::getDequantCoeff returns them (w*h int32, value 16 = neutral), back to
    back in one arena; 'off' maps (log2w, log2h) to the table's offset.  Low frequencies get smaller values, as typical lists do."""
    off, parts, o = {}, [], 0
    for l2w in range(1, 7):
        for l2h in range(1, 7):
            w, h = 1 << l2w, 1 << l2h
            yy, xx = np.mgrid[0:h, 0:w]
            t = 8 + ((xx * 8) // w + (yy * 8) // h) * int(rng.integers(1, 12)) + rng.integers(0, 4, size=(h, w))
            off[(l2w, l2h)] = o; parts.append(np.clip(t, 1, 255).astype(np.int32).reshape(-1)); o += w * h
    return dict(off=off, arena=np.concatenate(parts))


def noise_planes(rng, W, H, bit_depth=10, chroma=True, strides=None):
    """Stand-in prediction / reference pictures: smooth gradient + band-limited noise, clipped to the bit depth."""
    mx = (1 << bit_depth) - 1
    out = []
    for c in range(3 if chroma else 1):
        w, h = (W, H) if c == 0 else (W >> 1, H >> 1)
        st = strides[c] if strides else w
        yy, xx = np.mgrid[0:h, 0:w]
        base = (mx / 2) + (mx / 4) * np.sin(xx / (37.0 + 11 * c)) * np.cos(yy / (53.0 - 7 * c))
        n = rng.normal(0, mx / 40, size=(h // 4 + 2, w // 4 + 2))
        n = np.kron(n, np.ones((4, 4)))[:h, :w]
        fine = rng.integers(-8, 9, size=(h, w))
        p = np.zeros((h, st), np.int16)
        p[:, :w] = np.clip(base + n + fine, 0, mx).astype(np.int16)
        out.append(p)
    return out


LF_DTYPE = np.dtype([("qp", "i1", (3,)), ("bs", "u1"), ("len", "u1"), ("flags", "u1")])
LFSLICE_DTYPE = np.dtype([("beta", "i1", (3,)), ("tc", "i1", (3,)), ("disable", "u1"), ("rsv", "u1")])


def unit_maps(cus, W, H, cu_attr=None):
    """Paint per-4x4-unit maps from a CU list: TU id, TU width/height (TUs are the <=64 tiles of a CU), CU index."""
    W4, H4 = (W + 3) // 4, (H + 3) // 4
    tu_id = np.zeros((H4, W4), np.int32); tu_w = np.zeros((H4, W4), np.int16); tu_h = np.zeros((H4, W4), np.int16)
    cu_ix = np.zeros((H4, W4), np.int32)
    n = 0
    for i, (cx, cy, cw, ch) in enumerate(cus):
        cu_ix[cy // 4:(cy + ch) // 4, cx // 4:(cx + cw) // 4] = i
        for ty in range(cy, cy + ch, 64):
            for tx in range(cx, cx + cw, 64):
                tw, th = min(64, cw), min(64, ch)
                n += 1
                sl = (slice(ty // 4, (ty + th) // 4), slice(tx // 4, (tx + tw) // 4))
                tu_id[sl] = n; tu_w[sl] = tw; tu_h[sl] = th
    return tu_id, tu_w, tu_h, cu_ix


def gen_lf_grid(rng, cus, W, H, bit_depth=10, cu_intra=None, cu_qp=None, p_bs0=0.3):
    """LoopFilterParam rasters for a CU list, consistent with the geometry the way calcFilterStrengths
    (reference LoopFilter.cpp:495, xSetMaxFilterLengthPQFromTransformSizes :780) derives them:
    edges only at TU boundaries; luma max lengths 1/1 next to a <=4 block, else 7 (>=32) or 3 per side;
    chroma 'large' flag when both sides are >= 8 chroma samples; Bs 2 next to intra, else 1 or 0 at random."""
    ncu = len(cus)
    cu_intra = (rng.random(ncu) < 0.2) if cu_intra is None else cu_intra
    cu_qp = rng.integers(22, 45, size=ncu) if cu_qp is None else cu_qp
    tu_id, tu_w, tu_h, cu_ix = unit_maps(cus, W, H)
    H4, W4 = tu_id.shape
    out = []
    for d in (0, 1):
        g = np.zeros((H4, W4), LF_DTYPE)
        if d == 0:
            edge = np.zeros((H4, W4), bool); edge[:, 1:] = tu_id[:, 1:] != tu_id[:, :-1]
            szQ = tu_w; szP = np.zeros_like(tu_w); szP[:, 1:] = tu_w[:, :-1]
            cuP = np.zeros_like(cu_ix); cuP[:, 1:] = cu_ix[:, :-1]
        else:
            edge = np.zeros((H4, W4), bool); edge[1:, :] = tu_id[1:, :] != tu_id[:-1, :]
            szQ = tu_h; szP = np.zeros_like(tu_h); szP[1:, :] = tu_h[:-1, :]
            cuP = np.zeros_like(cu_ix); cuP[1:, :] = cu_ix[:-1, :]
        intra = cu_intra[cu_ix] | cu_intra[cuP]
        bsY = np.where(intra, 2, (rng.random((H4, W4)) >= p_bs0).astype(np.int64))
        bsU = np.where(intra, 2, (rng.random((H4, W4)) >= p_bs0).astype(np.int64))
        bsV = np.where(intra, 2, (rng.random((H4, W4)) >= p_bs0).astype(np.int64))
        bs = (bsY | (bsU << 2) | (bsV << 4)) * edge
        small = (szP <= 4) | (szQ <= 4)
        lenP = np.where(small, 1, np.where(szP >= 32, 7, 3)); lenQ = np.where(small, 1, np.where(szQ >= 32, 7, 3))
        qpl = (cu_qp[cu_ix] + cu_qp[cuP] + 1) >> 1
        g["bs"] = bs
        g["len"] = np.where(edge, 128 + (lenP << 4) + lenQ, 0)
        g["flags"] = np.where(edge & (szP >= 16) & (szQ >= 16), 32, 0) | (edge * 3)
        g["qp"][..., 0] = qpl
        g["qp"][..., 1] = np.clip(qpl - 1, 0, 63); g["qp"][..., 2] = np.clip(qpl + 1, 0, 63)
        out.append(np.ascontiguousarray(g))
    return out[0], out[1]


SAO_DTYPE = np.dtype([("type", "u1", (3,)), ("band", "u1", (3,)), ("offset", "i1", (3, 5)), ("avail", "u1"), ("rsv", "u1", (2,))])
ALFCTU_DTYPE = np.dtype([("enable", "u1", (3,)), ("lumaSet", "u1"), ("chromaAlt", "u1", (2,)), ("ccIdx", "u1", (2,))])
assert SAO_DTYPE.itemsize == 24 and ALFCTU_DTYPE.itemsize == 8
AV_L, AV_R, AV_A, AV_B, AV_AL, AV_AR, AV_BL, AV_BR = 1, 2, 4, 8, 16, 32, 64, 128


def picture_avail(ctusW, ctusH):
    """8-neighbour CTU availability when only the picture limits restrict it (single slice / tile)."""
    av = np.zeros((ctusH, ctusW), np.uint8)
    for y in range(ctusH):
        for x in range(ctusW):
            l, r, a, b = x > 0, x + 1 < ctusW, y > 0, y + 1 < ctusH
            av[y, x] = (AV_L * l | AV_R * r | AV_A * a | AV_B * b | AV_AL * (l and a) | AV_AR * (r and a)
                        | AV_BL * (l and b) | AV_BR * (r and b))
    return av.reshape(-1)


def gen_sao(rng, W, H, ctu=128, bit_depth=10, p_on=0.4, chroma=True):
    """Per-CTU SAO records (SURVEY §8d: SAO on 40 % of CTUs, EO:BO 3:1, offsets in [-7,7] scaled by 1<<max(0,bd-10))."""
    ctusW, ctusH = (W + ctu - 1) // ctu, (H + ctu - 1) // ctu
    n = ctusW * ctusH
    s = np.zeros(n, SAO_DTYPE)
    s["type"] = 255
    scale = 1 << max(0, bit_depth - 10)
    for i in range(n):
        for c in range(3 if chroma else 1):
            if rng.random() < p_on:
                t = int(rng.integers(0, 4)) if rng.random() < 0.75 else 4
                s["type"][i, c] = t
                off = rng.integers(-7, 8, size=5) * scale
                if t < 4: off[2] = 0
                s["offset"][i, c] = off
                s["band"][i, c] = int(rng.integers(0, 32))
    s["avail"] = picture_avail(ctusW, ctusH)
    return s


ALF_TR = [[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12], [9, 4, 10, 8, 1, 5, 11, 7, 3, 0, 2, 6, 12],
          [0, 3, 2, 1, 8, 7, 6, 5, 4, 9, 10, 11, 12], [9, 8, 10, 4, 3, 7, 11, 5, 1, 0, 2, 6, 12]]   # AdaptiveLoopFilter.cpp:97-112


def _fixed_sets():
    import os
    return np.load(os.path.join(os.path.dirname(__file__), "alf_fixed_sets.npy"))


def gen_alf(rng, W, H, ctu=128, bit_depth=10, n_aps=2, n_chroma_alts=3, n_cc=(2, 3), p_luma=0.8, p_chroma=0.6, p_cc=0.3):
    """ALF tables (16 fixed sets + n_aps random APS sets, pre-transposed like lumaCoeffFinal) and per-CTU controls."""
    clipv = [1 << bit_depth, 1 << (bit_depth - 3), 1 << (bit_depth - 5), 1 << (bit_depth - 7)]   # m_alfClippVls
    nsets = 16 + n_aps
    coef = np.zeros((nsets, 4, 25, 13), np.int16); clip = np.zeros((nsets, 4, 25, 13), np.int16)
    coef[:16] = _fixed_sets(); clip[:16] = clipv[0]
    for s in range(16, nsets):
        base = rng.integers(-40, 41, size=(25, 13)).astype(np.int16); base[:, 12] = 128
        bclip = rng.choice(clipv, size=(25, 13)).astype(np.int16)
        for t in range(4):
            coef[s, t] = base[:, ALF_TR[t]]; clip[s, t] = bclip[:, ALF_TR[t]]
    ccoef = rng.integers(-40, 41, size=(n_chroma_alts, 7)).astype(np.int16); ccoef[:, 6] = 128
    cclip = rng.choice(clipv, size=(n_chroma_alts, 7)).astype(np.int16)
    cclip[0, :] = clipv[0]                                      # first alternative without clipping (clip index 0), as encoders mostly signal
    cc = [rng.integers(-63, 64, size=(n_cc[c], 7)).astype(np.int16) for c in range(2)]
    ctusW, ctusH = (W + ctu - 1) // ctu, (H + ctu - 1) // ctu
    n = ctusW * ctusH
    a = np.zeros(n, ALFCTU_DTYPE)
    a["enable"][:, 0] = rng.random(n) < p_luma
    a["enable"][:, 1] = rng.random(n) < p_chroma; a["enable"][:, 2] = rng.random(n) < p_chroma
    a["lumaSet"] = rng.integers(0, nsets, size=n)
    a["chromaAlt"] = rng.integers(0, n_chroma_alts, size=(n, 2))
    for c in range(2):
        a["ccIdx"][:, c] = np.where(rng.random(n) < p_cc, rng.integers(1, n_cc[c] + 1, size=n), 0) if n_cc[c] else 0
    return dict(lumaCoeff=np.ascontiguousarray(coef), lumaClip=np.ascontiguousarray(clip), chromaCoeff=ccoef, chromaClip=cclip,
                cc=cc, ctus=a)


PU_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("w", "u1"), ("h", "u1"), ("flags", "u1"), ("bcwW1", "i1"), ("refSlot", "i1", (2,)),
                     ("interDir", "u1"), ("wpIdx", "u1"), ("dmvrOff", "<u4"), ("mv", "<i4", (2, 2)), ("cpmv", "<i4", (2, 2, 2))])
assert PU_DTYPE.itemsize == 64
PU_BDOF, PU_DMVR, PU_ALTHPEL, PU_AFFINE, PU_AFFINE6, PU_PROF0, PU_PROF1, PU_GEO = 1, 2, 4, 8, 16, 32, 64, 128


def gen_pus(rng, cus, W, H, p_inter=1.0, p_bi=0.6, p_dmvr=0.35, p_bdof=0.35, p_affine=0.12, p_bcw=0.15, mv_sigma=6.0, p_int_mv=0.15, p_prof=1.0, p_geo=0.0):
    """Inter PU records for a CU list (SURVEY §8d: MVs ~ N(0, 6 px) in 1/16 units; refs from 4 DPB slots:
    list 0 = {0, 1}, list 1 = {2, 3}; (0,2) and (1,3) are the equal-POC-distance pairs that allow BDOF / DMVR)."""
    recs = []
    dmvr_off = 0
    for (x, y, w, h) in cus:
        if w > 128 or h > 128 or rng.random() >= p_inter:
            continue
        r = np.zeros((), PU_DTYPE)
        r["x"], r["y"], r["w"], r["h"] = x, y, w, h
        r["bcwW1"] = 4
        mv = np.rint(rng.normal(0, mv_sigma * 16, size=(2, 2))).astype(np.int64)
        if rng.random() < p_int_mv: mv = (mv >> 4) << 4
        if rng.random() < 0.1: mv[:, rng.integers(0, 2)] &= ~15                      # one integer component
        if rng.random() < 0.03: mv += rng.integers(-3000, 3000, size=(2, 2))          # far outside the picture -> clipMv
        r["mv"] = mv
        if p_geo and 8 <= w <= 64 and 8 <= h <= 64 and w < 8 * h and h < 8 * w and rng.random() < p_geo:
            # geometric partitioning: two uni-predicted partitions (any slots, also from the same list), split direction in bcwW1
            r["refSlot"] = (int(rng.integers(0, 4)), int(rng.integers(0, 4))); r["interDir"] = 3
            r["bcwW1"] = int(rng.integers(0, 64)); r["flags"] = PU_GEO
            if w >= 8 and h >= 8 and w * h >= 128:
                r["dmvrOff"] = dmvr_off; dmvr_off += max(1, w >> 4) * max(1, h >> 4)
            recs.append(r); continue
        can_bi = (w + h) > 12
        bi = can_bi and rng.random() < p_bi
        big = w >= 8 and h >= 8 and w * h >= 128
        flags = 0
        if bi:
            u = rng.random()
            if big and u < p_dmvr:
                pair = int(rng.integers(0, 2)); r["refSlot"] = (pair, 2 + pair)
                flags |= PU_DMVR | (PU_BDOF if rng.random() < 0.8 else 0)
            elif big and u < p_dmvr + p_bdof:
                pair = int(rng.integers(0, 2)); r["refSlot"] = (pair, 2 + pair)
                flags |= PU_BDOF
            else:
                r["refSlot"] = (int(rng.integers(0, 2)), 2 + int(rng.integers(0, 2)))
                if w * h >= 256 and rng.random() < p_bcw: r["bcwW1"] = int(rng.choice([-2, 3, 5, 10]))
            r["interDir"] = 3
        else:
            l = int(rng.integers(0, 2))
            r["refSlot"] = (int(rng.integers(0, 2)), -1) if l == 0 else (-1, 2 + int(rng.integers(0, 2)))
            r["interDir"] = 1 + l
        if not (flags & (PU_DMVR | PU_BDOF)) and w >= 8 and h >= 8 and rng.random() < p_affine:
            flags |= PU_AFFINE | (PU_AFFINE6 if rng.random() < 0.5 else 0)
            if rng.random() < p_prof: flags |= PU_PROF0 | PU_PROF1   # PROF is a sequence/picture-level switch (sps_prof / ph_prof_disabled)
            big_d = rng.random() < 0.15
            for l in range(2):
                d = rng.integers(-400, 401, size=(2, 2)) if big_d else rng.integers(-24, 25, size=(2, 2))
                if rng.random() < 0.1: d[:] = 0
                r["cpmv"][l] = mv[l] + d
        elif not (flags & PU_DMVR) and rng.random() < 0.1:
            flags |= PU_ALTHPEL
        if big:
            r["dmvrOff"] = dmvr_off
            dmvr_off += max(1, w >> 4) * max(1, h >> 4)
        r["flags"] = flags
        recs.append(r)
    pus = np.array(recs, PU_DTYPE) if recs else np.zeros(0, PU_DTYPE)
    return pus, dmvr_off


WP_DTYPE = np.dtype([("w0", "<i2", (3,)), ("w1", "<i2", (3,)), ("offset", "<i2", (3,)), ("shift", "u1", (3,)), ("rsv", "u1", (3,))])
assert WP_DTYPE.itemsize == 24


def gen_wp(rng, bit_depth, pus):
    """Explicit weighted prediction for a B picture with pps_weighted_bipred: random (log2WeightDenom, iWeight, iOffset) per
    (list, refIdx, component) as a slice header carries them, the b200_wp entries WeightPrediction::getWpScaling (reference
    WeightPrediction.cpp:67-147) derives for every (refIdx0, refIdx1) combination, and pus['wpIdx'] set for the PUs they apply to
    (BcwIdx == default, InterPrediction.cpp:733).  Returns (raw int32 [2][2][3][3], entries)."""
    raw = np.zeros((2, 2, 3, 3), np.int32)
    den = [int(rng.integers(0, 8)), int(rng.integers(0, 8))]          # luma_log2_weight_denom, chroma
    for l in range(2):
        for i in range(2):
            for c in range(3):
                d = den[0] if c == 0 else den[1]
                plain = rng.random() < 0.25
                raw[l, i, c] = (d, (1 << d) if plain else (1 << d) + int(rng.integers(-128, 128)), 0 if plain else int(rng.integers(-128, 128)))
    sc = 1 << (bit_depth - 8)
    ent = np.zeros(8, WP_DTYPE); idx = {}
    k = 0
    for r0 in (-1, 0, 1):
        for r1 in (-1, 0, 1):
            if r0 < 0 and r1 < 0: continue
            e = ent[k]
            for c in range(3):
                if r0 >= 0 and r1 >= 0:
                    e["w0"][c] = raw[0, r0, c, 1]; e["w1"][c] = raw[1, r1, c, 1]
                    e["offset"][c] = (raw[0, r0, c, 2] + raw[1, r1, c, 2]) * sc; e["shift"][c] = raw[0, r0, c, 0] + 1
                else:
                    l, r = (0, r0) if r0 >= 0 else (1, r1)
                    e["w0"][c] = raw[l, r, c, 1]; e["offset"][c] = raw[l, r, c, 2] * sc; e["shift"][c] = raw[l, r, c, 0]
            idx[(r0, r1)] = k + 1; k += 1
    for p in pus:
        r0 = -1 if p["refSlot"][0] < 0 else int(p["refSlot"][0]) & 1
        r1 = -1 if p["refSlot"][1] < 0 else int(p["refSlot"][1]) & 1
        p["wpIdx"] = idx[(r0, r1)] if p["bcwW1"] == 4 and not (p["flags"] & PU_GEO) else 0    # GEO never combines with explicit weights (xPredInterBi :731)
    return raw, ent


LMCS_VPDU_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("availLeft", "u1"), ("availAbove", "u1")])


def lmcs_tables(bit_depth, min_bin, max_bin, delta_cw, chr_offset):
    """Reshape::constructReshaper (reference CommonLib/Reshape.cpp:317-373) restated for the generator: code-word deltas of the LMCS
    APS -> pivots, forward scale, chroma-scale LUT, inverse LUT.  tests/test_lmcs_oracle_vs_ref.py checks it against the real class."""
    FP = 11
    n = 1 << bit_depth; org = n // 16; l2 = org.bit_length() - 1
    bin_cw = [0] * 16
    for i in range(min_bin, max_bin + 1): bin_cw[i] = delta_cw[i] + org
    piv = [0] * 17; inp = [0] * 17; fwd = [0] * 16; inv = [0] * 16; cadj = [1 << FP] * 16
    for i in range(16):
        piv[i + 1] = piv[i] + bin_cw[i]; inp[i + 1] = inp[i] + org
        fwd[i] = (bin_cw[i] * (1 << FP) + (1 << (l2 - 1))) >> l2
        if bin_cw[i]:
            inv[i] = org * (1 << FP) // bin_cw[i]; cadj[i] = org * (1 << FP) // (bin_cw[i] + chr_offset)
    lut = np.zeros(n, np.int16)
    for v in range(n):
        idx = min_bin
        while idx <= max_bin and not v < piv[idx + 1]: idx += 1
        idx = min(idx, 15)
        lut[v] = min(max(inp[idx] + ((inv[idx] * (v - piv[idx]) + (1 << (FP - 1))) >> FP), 0), n - 1)
    return dict(orgCW=org, reshapePivot=piv, inputPivot=inp, fwdScaleCoef=fwd, chromaAdjHelpLUT=cadj, invLUT=lut)


def gen_lmcs(rng, bit_depth, cus, W, H, ctu, chroma_adj=True):
    """A legal random LMCS model (code words are multiples of 1 << (bd-5), so the pivot constraint of Reshape.cpp:355-363 holds) and the
    per-VPDU records: position of the CU covering each VPDU's top-left sample, neighbours available inside the picture (one slice, one tile)."""
    org = (1 << bit_depth) // 16; step = 1 << (bit_depth - 5)
    min_bin = int(rng.integers(0, 3)); max_bin = int(rng.integers(12, 16))
    while True:
        cw = rng.integers(1, 5, size=16) * step            # 0.5x .. 2x of the identity code word
        if int(cw[min_bin:max_bin + 1].sum()) <= (1 << bit_depth) - 1: break
    delta = [int(cw[i]) - org if min_bin <= i <= max_bin else 0 for i in range(16)]
    # lmcsCW[i] + lmcsDeltaCrs must stay in [OrgCW >> 3, (OrgCW << 3) - 1] (Reshape.cpp:332-333)
    chr_off = int(rng.integers(max(-7, (org >> 3) - int(cw[min_bin:max_bin + 1].min())), 8)) if chroma_adj else 0
    return _lmcs_dict(bit_depth, min_bin, max_bin, delta, chr_off, chroma_adj, lmcs_vpdu_records(cus, W, H, ctu))


def lmcs_vpdu_records(cus, W, H, ctu):
    """The b200_lmcs_vpdu raster of a CU list: the origin of the CU covering each VPDU's top-left sample, neighbours available inside the picture
    (one slice, one tile)."""
    vs = 64 if ctu == 128 else ctu
    vW, vH = (W + vs - 1) // vs, (H + vs - 1) // vs
    owner = np.zeros(((H + 3) // 4, (W + 3) // 4), np.int32)         # CU lookup on the 4x4 grid
    for i, (x, y, w, h) in enumerate(cus): owner[y // 4:(y + h) // 4, x // 4:(x + w) // 4] = i
    vp = np.zeros(vW * vH, LMCS_VPDU_DTYPE)
    for j in range(vH):
        for i in range(vW):
            x, y, w, h = cus[owner[j * vs // 4, i * vs // 4]]
            vp[j * vW + i] = (x, y, x > 0, y > 0)
    return vp


def _lmcs_dict(bit_depth, min_bin, max_bin, delta, chr_off, chroma_adj, vp):
    from . import abi as A
    t = lmcs_tables(bit_depth, min_bin, max_bin, delta, chr_off)
    L = A.Lmcs(); L.chromaAdj = int(chroma_adj); L.minBinIdx = min_bin; L.maxBinIdx = max_bin; L.orgCW = t["orgCW"]
    for i in range(17): L.reshapePivot[i] = t["reshapePivot"][i]; L.inputPivot[i] = t["inputPivot"][i]
    for i in range(16): L.fwdScaleCoef[i] = t["fwdScaleCoef"][i]; L.chromaAdjHelpLUT[i] = t["chromaAdjHelpLUT"][i]
    L.invLUT = t["invLUT"].ctypes.data; L.vpdus = vp.ctypes.data
    return dict(struct=L, invLUT=t["invLUT"], vpdus=vp, minBin=min_bin, maxBin=max_bin, delta=delta, chrOff=chr_off, tables=t)


# ---- LMCS: designed models and pictures (tests/test_lmcs_*.py)
LMCS_MODELS = ("identity", "compress", "expand_max", "fine_pivots", "narrow_bins", "single_bin", "full_bins", "crs_min", "crs_max")


def lmcs_model_problems(bit_depth, min_bin, max_bin, delta, chr_off):
    """The conformance checks of Reshape::constructReshaper (reference CommonLib/Reshape.cpp:331-363) and the APS syntax ranges: a list of the broken
    rules, empty for a legal model."""
    org = (1 << bit_depth) // 16; lo, hi, s = org >> 3, (org << 3) - 1, bit_depth - 5
    out = []
    if not 0 <= min_bin <= max_bin <= 15: return ["0 <= minBin <= maxBin <= 15"]
    if not -7 <= chr_off <= 7: out.append("lmcsDeltaCrs outside -7..7")
    cw = [delta[i] + org if min_bin <= i <= max_bin else 0 for i in range(16)]
    for i in range(min_bin, max_bin + 1):
        if not lo <= cw[i] <= hi: out.append(f"lmcsCW[{i}] = {cw[i]} outside {lo}..{hi}")
        if not lo <= cw[i] + chr_off <= hi: out.append(f"lmcsCW[{i}] + lmcsDeltaCrs = {cw[i] + chr_off} outside {lo}..{hi}")
    if sum(cw) > (1 << bit_depth) - 1: out.append(f"sum of code words {sum(cw)} above 2^bd - 1")
    piv = [0]
    for c in cw: piv.append(piv[-1] + c)
    for i in range(min_bin, max_bin + 1):
        if piv[i] % (1 << s) and piv[i] >> s == piv[i + 1] >> s: out.append(f"pivot rule at bin {i} (LmcsPivot {piv[i]} -> {piv[i + 1]})")
    return out


def _lmcs_design(name, bd):
    """(minBin, maxBin, code words of bins minBin..maxBin, chroma offset) of a designed model.  A bin that starts off the 1 << (bd - 5) grid is raised
    until it reaches the next grid line (the pivot rule, Reshape.cpp:355-363)."""
    org = (1 << bd) // 16; step = 1 << (bd - 5); lo, hi = org >> 3, (org << 3) - 1
    mn, mx, tg, off = {
        "identity": (0, 14, [org] * 15, 0),                              # all 16 bins at OrgCW would sum to 2^bd, one above the limit
        "compress": (0, 15, [org, step, org - 1, step + 1] * 4, 0),       # every code word <= OrgCW: the inverse map expands
        "expand_max": (1, 14, [lo] * 6 + [hi] + [lo] * 7, 0),             # one bin at (OrgCW << 3) - 1, the rest at OrgCW >> 3 (raised by the pivot rule)
        "fine_pivots": (0, 15, [step + 3, step - 1, org - 3, step + 1] * 4, 0),
        "narrow_bins": (5, 9, [2 * org, org + step, org, 3 * step, org - step], 0),
        "single_bin": (7, 7, [3 * org], 0),
        "full_bins": (0, 15, [org + step, org - step] * 7 + [org, org - step], 0),
        "crs_min": (2, 13, [lo + 7, org, org, org] * 3, -7),             # lmcsCW + lmcsDeltaCrs = OrgCW >> 3 in bins 2, 6, 10: chroma scale 16384
        "crs_max": (4, 11, [org] * 3 + [hi - 7] + [org] * 4, 7),          # lmcsCW + lmcsDeltaCrs = (OrgCW << 3) - 1 in bin 7
    }[name]
    cw, p = [], 0
    for t in tg:
        if p % step: t = max(t, step - p % step)
        cw.append(t); p += t
    return mn, mx, cw, off


def lmcs_model(name, bd, chroma_adj=True, vpdus=None):
    """A designed LMCS model (LMCS_MODELS) at bit depth bd, in the dict gen_lmcs returns; vpdus: its b200_lmcs_vpdu raster (default: one record)."""
    mn, mx, cw, off = _lmcs_design(name, bd)
    org = (1 << bd) // 16
    delta = [cw[i - mn] - org if mn <= i <= mx else 0 for i in range(16)]
    d = _lmcs_dict(bd, mn, mx, delta, off if chroma_adj else 0, chroma_adj, np.zeros(1, LMCS_VPDU_DTYPE) if vpdus is None else vpdus)
    d["name"] = name
    return d


def lmcs_fwd(m, v):
    """The forward map (rspFwdCore, reference CommonLib/Buffer.cpp:321) of an array of samples under model dict m, before its clip to 0..2^bd - 1."""
    t = m["tables"]; l2 = int(t["orgCW"]).bit_length() - 1
    v = np.asarray(v, np.int64); idx = v >> l2
    piv, inp, fwd = (np.array(t[k], np.int64) for k in ("reshapePivot", "inputPivot", "fwdScaleCoef"))
    return piv[idx] + ((fwd[idx] * (v - inp[idx]) + (1 << 10)) >> 11)


def lmcs_targets(m, bd):
    """The VPDU neighbour averages the sweep aims at for model m: pivot - 1, pivot and pivot + 1 of every bin boundary minBin..maxBin + 1, 0 (below the
    model's range) and 2^bd - 1 (above it), inside 0..2^bd - 1."""
    piv = m["tables"]["reshapePivot"]; pmax = (1 << bd) - 1
    t = {0, pmax}
    for k in range(m["minBin"], m["maxBin"] + 2):
        t |= {piv[k] - 1, piv[k], piv[k] + 1}
    return sorted(v for v in t if 0 <= v <= pmax)


def lmcs_vpdu_walk(v, W, H, ctu):
    """The luma positions lmcs_vpdu_kernel sums for one VPDU record, with multiplicity (the clamps at the picture's last row / column repeat a sample):
    dict (y, x) -> count, and the number of samples (0, n or 2n)."""
    nn = min(64, ctu); x, y = int(v["x"]), int(v["y"])
    pos = {}
    for i in range(nn):
        if v["availLeft"]: k = H - y - 1 if y + i >= H else i; pos[(y + k, x - 1)] = pos.get((y + k, x - 1), 0) + 1
        if v["availAbove"]: k = W - x - 1 if x + i >= W else i; pos[(y - 1, x + k)] = pos.get((y - 1, x + k), 0) + 1
    return pos, nn * (int(bool(v["availLeft"])) + int(bool(v["availAbove"])))


def lmcs_average(luma, v, W, H, ctu, bd):
    """The rounded neighbour average lmcs_vpdu_kernel derives for a record (1 << (bd - 1) without neighbours)."""
    pos, n = lmcs_vpdu_walk(v, W, H, ctu)
    if not n: return 1 << (bd - 1)
    l2 = n.bit_length() - 1
    return (sum(int(luma[p]) * c for p, c in pos.items()) + (n >> 1)) >> l2


def _lmcs_place_averages(luma, vp, W, H, ctu, bd, targets):
    """Writes the neighbourhood samples of the records in raster order so that their rounded averages take the values of `targets` (each once while
    any is left, the ones farthest from mid-grey first, then again from the start).  Walks share samples (a VPDU's bottom-right sample is in the walks
    of two later VPDUs), so a record takes the first target still reachable with the samples earlier records fixed."""
    pmax = (1 << bd) - 1; fixed = set(); seen = set()
    order = sorted(targets, key=lambda t: -abs(2 * t - pmax))
    todo = list(order)
    for v in vp:
        key = (int(v["x"]), int(v["y"]))
        pos, n = lmcs_vpdu_walk(v, W, H, ctu)
        if not n or key in seen: continue                              # no neighbours, or a CU whose walk an earlier VPDU already set
        seen.add(key)
        free = sorted((p for p in pos if p not in fixed), key=lambda p: -pos[p])
        have = sum(int(luma[p]) * c for p, c in pos.items() if p in fixed)
        for t in (todo or order):
            rest, left = t * n - have, sum(pos[p] for p in free)       # the rounded average is t for sums t * n - n/2 .. t * n + n/2 - 1
            for p in free:                                              # spread the rest evenly; the last samples absorb the rounding
                c = pos[p]; val = min(pmax, max(0, (rest + left // 2) // left))
                luma[p] = val; rest -= val * c; left -= c
            if lmcs_average(luma, v, W, H, ctu, bd) == t:
                if t in todo: todo.remove(t)
                break
        fixed |= set(free)


# (kind, model, bit depth, variant) of every case; names "kind_model_Nbit[_variant]"
def _lmcs_sweep_cases():
    out = {}
    for bd in (8, 10, 12):
        for m in LMCS_MODELS:
            for st in ("stride8", "odd"): out[f"inverse_{m}_{bd}bit_{st}"] = ("inverse", m, bd, st)
        for m in ("compress", "expand_max"): out[f"forward_{m}_{bd}bit"] = ("forward", m, bd, None)
        out[f"vpdu_full_bins_{bd}bit_ctu32"] = ("vpdu", "full_bins", bd, "ctu32")
        out[f"vpdu_single_bin_{bd}bit_ctu64"] = ("vpdu", "single_bin", bd, "ctu64")
        out[f"vpdu_single_bin_{bd}bit_ctu128"] = ("vpdu", "single_bin", bd, "ctu128")
        for adj in ("adj", "noadj"): out[f"yuv400_fine_pivots_{bd}bit_{adj}"] = ("yuv400", "fine_pivots", bd, adj)
    out["extremes_crs_min_12bit"] = ("extremes", "crs_min", 12, None)
    return out


LMCS_SWEEP = _lmcs_sweep_cases()
# CU rectangles of the VPDU cases: one CU per CTU at CTU 32 / 64 (the reference arm's structure); at CTU 128 a 128x128 CU and 64x128 CUs that
# cover several VPDUs, and CUs whose walks reach past the picture's last row / column
_LMCS_VPDU_GEOM = {
    "ctu32": (256, 384, 32, None),
    "ctu64": (200, 136, 64, None),
    "ctu128": (232, 120, 128, [(0, 0, 128, 128), (128, 0, 64, 128), (192, 0, 32, 64), (224, 0, 32, 64), (192, 64, 64, 64)]),
}


def _lmcs_ramp(W, H, bd, shift=0):
    yy, xx = np.mgrid[0:H, 0:W]
    return ((yy * W + xx + shift) % (1 << bd)).astype(np.int16)


def _lmcs_case(name):
    from . import abi as A
    import ctypes as C, zlib
    kind, model, bd, var = LMCS_SWEEP[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    pmax, mid = (1 << bd) - 1, 1 << (bd - 1)
    chroma = kind != "yuv400"
    cus, pus, tus, coefs, tags = None, np.zeros(0, PU_DTYPE), np.zeros(0, A.TU_DTYPE), np.zeros(1, np.int16), []
    if kind == "inverse":                                               # a ramp of every value as `given` luma: the output is invLUT[v]
        W, H, ctu = 64, 64, 64
        strides = (64, 32, 32) if var == "stride8" else (67, 35, 35)
        given = [np.full((H, strides[0]), -7, np.int16)] + [np.full((H // 2, strides[c]), -7, np.int16) for c in (1, 2)]
        given[0][:, :W] = _lmcs_ramp(W, H, bd); given[1][:, :W // 2] = mid; given[2][:, :W // 2] = mid // 2
    elif kind == "vpdu":
        W, H, ctu, cus = _LMCS_VPDU_GEOM[var]
        strides = None
    elif kind == "extremes":
        W, H, ctu, strides = 128, 128, 32, None
    else:
        W, H, ctu, strides = 64, 64, 64, None
    if cus is None: cus = [(x, y, min(ctu, W - x), min(ctu, H - y)) for y in range(0, H, ctu) for x in range(0, W, ctu)]
    vp = lmcs_vpdu_records(cus, W, H, ctu)
    m = lmcs_model(model, bd, chroma_adj=var != "noadj", vpdus=vp)
    g = A.make_geom(W, H, bd, chroma_format=1 if chroma else 0, ctu=ctu, strides=strides)
    dpb = [noise_planes(rng, W, H, bd, strides=strides) for _ in range(4)]
    if kind in ("forward", "yuv400"):
        # the ramp in slot 0, copied by zero-MV uni PUs of several sizes and by one bi PU whose two references are slot 0 (integer MVs: the bi average of
        # two equal predictions is exact); no DMVR / BDOF, no residual on the forward cases
        dpb[0][0][:] = _lmcs_ramp(W, H, bd, shift=17)
        rects = [(0, 0, 32, 32, "bi")] + [(32 + 16 * (i % 2), 16 * (i // 2), 16, 16, "uni") for i in range(4)] + \
                [(0, 32 + 8 * j, 32, 8, "uni") for j in range(2)] + [(8 * i, 48, 8, 16, "uni") for i in range(4)] + \
                [(32 + 8 * (i % 4), 32 + 8 * (i // 4), 8, 8, "uni") for i in range(16)]
        pus = np.zeros(len(rects), PU_DTYPE)
        for r, (x, y, w, h, kd) in zip(pus, rects):
            r["x"], r["y"], r["w"], r["h"], r["bcwW1"] = x, y, w, h, 4
            if kd == "bi": r["refSlot"] = (0, 0); r["interDir"] = 3
            else: r["refSlot"] = (0, -1); r["interDir"] = 1
            tags.append(f"{kd} PU {w}x{h} at ({x}, {y})")
        given = None
        if kind == "yuv400":                                            # luma TUs on top: residual added in the mapped domain
            b = _K1Case(W, bd, rng)
            ts = dict(flags=A.TU_TS, qp=4 - 6 * (bd - 8))
            for k, (x, y) in enumerate([(0, 0), (8, 8), (40, 40), (56, 0)]):
                b.add(f"luma TS 8x8 at ({x}, {y})", 0, 8, 8, rng.integers(-pmax // 4, pmax // 4 + 1, (8, 8)), at=(x, y), **ts)
            tus, coefs = np.array(b.recs, A.TU_DTYPE), np.concatenate(b.levels); tags += b.tags
    else:
        if kind != "inverse":                                           # designed luma neighbourhoods + chroma TUs that show each VPDU's scale
            luma = np.full((H, W), mid, np.int16)
            vs = 64 if ctu == 128 else ctu
            if kind == "extremes":                                      # every average inside a bin whose chroma scale is 16384
                piv = m["tables"]["reshapePivot"]; bins = [i for i in range(16) if m["tables"]["chromaAdjHelpLUT"][i] == 16384]
                targets = [piv[b] + k for b in bins for k in range(3)]
            else:
                targets = lmcs_targets(m, bd)
            _lmcs_place_averages(luma, vp, W, H, ctu, bd, targets)
            given = [luma, np.full((H // 2, W // 2), mid, np.int16), np.full((H // 2, W // 2), mid, np.int16)]
            b = _K1Case(W, bd, rng)
            ts = dict(flags=A.TU_TS, qp=4 - 6 * (bd - 8))
            vW = (W + vs - 1) // vs
            for k, v in enumerate(vp):
                cx, cy = (k % vW) * vs // 2, (k // vW) * vs // 2
                cw, ch = min(vs // 2, W // 2 - cx), min(vs // 2, H // 2 - cy)
                R = [1 << bd, -(1 << bd), 4095, -4096][k % 4] if kind == "extremes" else (37 + 11 * k) % (mid // 2) + 5
                big = 8 if min(cw, ch) >= 8 else 4
                b.add(f"VPDU {k} Cb DC {big}x{big}", 1, big, big, np.full((big, big), R), at=(cx, cy), **ts)
                b.add(f"VPDU {k} Cr DC {big}x{big}", 2, big, big, np.full((big, big), -R), at=(cx, cy), **ts)
                if cw >= big + 4 and ch >= 4:
                    ict = (1, -1, 2, -2, 3, -3)[k % 6]
                    b.add(f"VPDU {k} joint CbCr 4x4 ict {ict}", 1 + (abs(ict) == 3), 4, 4, np.full((4, 4), R), at=(cx + big, cy), ict=ict, **ts)
                if ch >= big + 2:
                    b.add(f"VPDU {k} Cb 2x2 (4 samples, unscaled)", 1, 2, 2, np.full((2, 2), R), at=(cx, cy + big), **ts)
                    b.add(f"VPDU {k} Cr 2x2 (4 samples, unscaled)", 2, 2, 2, np.full((2, 2), -R), at=(cx, cy + big), **ts)
            tus, coefs = np.array(b.recs, A.TU_DTYPE), np.concatenate(b.levels); tags += b.tags
    if not chroma:
        g.stride[1] = g.stride[2] = 0
        dpb = [[p[0], np.zeros((H // 2, W // 2), np.int16), np.zeros((H // 2, W // 2), np.int16)] for p in dpb]
    p = A.Picture(); p.dstSlot = 4; p.flags = A.PIC_LMCS; p.lmcs = C.addressof(m["struct"])
    d = dict(pus=pus, ndmvr=0, tus=tus, coefs=coefs, lmcs=m)
    p.pus = pus.ctypes.data; p.numPus = len(pus); p.numDmvr = 1
    p.tus = tus.ctypes.data; p.numTus = len(tus); p.coefs = coefs.ctypes.data; p.numCoefs = len(coefs)
    if given is not None:
        d["given"] = given
        for c in range(3 if chroma else 1): p.given[c] = given[c].ctypes.data
    d["struct"] = p
    return dict(name=name, kind=kind, model=model, bd=bd, variant=var, g=g, W=W, H=H, ctu=ctu, chroma=chroma, strides=strides, cus=cus, dpb=dpb,
                pic=d, tags=tags)


def lmcs_sweep(name):
    """One case of the designed LMCS sweep (LMCS_SWEEP): geometry (g, W, H, bd, ctu, chroma, strides), CU rectangles, DPB slots (4 x [Y, Cb, Cr]), the
    picture dict (pic: pus, tus, coefs, given, lmcs = the model dict, struct = the b200_picture, destination slot 4, filters off) and per-record tags.
    inverse: a ramp of every value as `given` luma, no PUs / TUs; forward: the ramp copied by zero-MV uni and bi PUs; vpdu: designed neighbour averages
    and one DC chroma TU per VPDU (with 4-sample and joint-CbCr TUs); extremes: residuals of +-2^bd scaled by 16384 at 12 bit; yuv400: 4:0:0 with
    PUs and luma TUs, chroma scaling on / off."""
    return _lmcs_case(name)


def gen_picture(rng, W, H, bit_depth=10, ctu=128, dst_slot=0, cu_kw=None, pu_kw=None, tu_kw=None, sao_p=0.4, alf_kw=None,
                deblock=True, sao=True, alf=True, lmcs=False, lmcs_chroma=True, wp=False, inter=True, given=None, cu_intra=None, intra_frac=0.0, p_ciip=0.25):
    """One synthetic post-parse picture (SURVEY §8d config 2/3): partition -> inter PUs (all CUs inter: intra-coded samples would
    be 'given' pixels, see DESIGN.md) -> TUs/levels -> deblocking grids -> SAO / ALF CTU parameters.
    Returns a dict of numpy arrays (kept alive by the caller) plus `struct`, the abi.Picture that points into them."""
    from . import abi as A
    import ctypes as C
    if intra_frac > 0:
        # intra CUs on the device (K6): CUs in decoding order, at most 64x64 (one TU per component); a fraction of them intra, the others inter.
        # Intra CUs: TUs flagged TU_RESI (residual -> residual planes) + b200_intra_tu records with ADD_RESI where a TU carries a residual.
        cus = gen_intra_layout(rng, W, H, ctu, **({"min_size": 8} | (cu_kw or {})))
        is_intra = rng.random(len(cus)) < intra_frac
        inter_cus = [cu for cu, f in zip(cus, is_intra) if not f]; intra_cus = [cu for cu, f in zip(cus, is_intra) if f]
        pus, ndmvr = gen_pus(rng, inter_cus, W, H, **(pu_kw or {})) if inter_cus else (np.zeros(0, PU_DTYPE), 0)
        tkw = {"p_cbf": 0.35, "p_intra": 0.0, "p_lfnst": 0.0, "p_bdpcm": 0.0} | (tu_kw or {})
        tus0, coefs0 = gen_tus(rng, inter_cus, bit_depth, **tkw)
        tus1, coefs1 = gen_tus(rng, intra_cus, bit_depth, **(tkw | {"p_intra": 1.0, "p_cbf": 0.6, "p_lfnst": 0.15, "p_bdpcm": 0.05}))
        tus1["coefOff"] += len(coefs0); tus1["flags"] |= A.TU_RESI
        tus, coefs = np.concatenate([tus0, tus1]), np.concatenate([coefs0, coefs1])
        # CIIP: plain merge-like inter CUs (no BDOF / DMVR / affine / GEO / BCW, at least 64 samples) also get a planar intra block that is blended
        # with their inter prediction; the weight counts the intra CUs left (at the bottom-left corner) and above (at the top-right corner)
        cu_idx = np.full(((H + 3) // 4, (W + 3) // 4), -1, np.int64)
        for i, (x, y, w, h) in enumerate(cus): cu_idx[y // 4:(y + h) // 4, x // 4:(x + w) // 4] = i
        inter_index = [i for i, f in enumerate(is_intra) if not f]
        ciip = {}
        for j, pu in enumerate(pus):
            i = inter_index[j]; x, y, w, h = cus[i]
            if pu["flags"] == 0 and pu["bcwW1"] == 4 and w * h >= 64 and rng.random() < p_ciip:
                nl = cu_idx[(y + h - 1) // 4, x // 4 - 1] if x > 0 else -1; na = cu_idx[y // 4 - 1, (x + w - 1) // 4] if y > 0 else -1
                ciip[i] = 3 - (0 if nl >= 0 and is_intra[nl] else 1) - (0 if na >= 0 and is_intra[na] else 1)
        ciip_cus = [cus[i] for i in sorted(ciip)]
        tus2, coefs2 = gen_tus(rng, ciip_cus, bit_depth, **(tkw | {"p_cbf": 0.6}))
        tus2["coefOff"] += len(coefs0) + len(coefs1)
        for t in tus2:                                              # chroma narrower than 4 has no CIIP block (predBlendIntraCiip :891): plain inter reconstruction there
            if not (t["comp"] and (1 << int(t["log2w"])) <= 2): t["flags"] |= A.TU_RESI
        # the plain inter TUs generated above for CIIP CUs are dropped: their residual goes through K6
        ciip_pos = {(x, y) for (x, y, w, h) in ciip_cus}
        keep = np.array([((int(t["x"]) << (1 if t["comp"] else 0), int(t["y"]) << (1 if t["comp"] else 0)) not in ciip_pos) for t in tus0], bool) if len(tus0) else np.zeros(0, bool)
        tus0 = tus0[keep]
        tus, coefs = np.concatenate([tus0, tus1, tus2]), np.concatenate([coefs0, coefs1, coefs2])
        mask = is_intra.copy()
        for i in ciip: mask[i] = True
        irecs = gen_intra_records(rng, cus, W, H, only=mask, p_lm=0.2, colloc=int(rng.integers(0, 2)), ciip=ciip, ctu=ctu)
        coded = set()
        for t in np.concatenate([tus1, tus2[(tus2["flags"] & A.TU_RESI) != 0]]):
            coded.add((int(t["comp"]), int(t["x"]), int(t["y"]))); 
            if t["ict"]: coded.add((3 - int(t["comp"]), int(t["x"]), int(t["y"])))
        for r in irecs:
            if (int(r["comp"]), int(r["x"]), int(r["y"])) in coded: r["flags"] |= A.INTRA_ADD_RESI
        if cu_intra is None: cu_intra = is_intra
    else:
        cus = partition(rng, W, H, ctu=ctu, **(cu_kw or {}))
        pus, ndmvr = gen_pus(rng, cus, W, H, **(pu_kw or {})) if inter else (np.zeros(0, PU_DTYPE), 0)
        tus, coefs = gen_tus(rng, cus, bit_depth, **({"p_cbf": 0.35, "p_intra": 0.0, "p_lfnst": 0.0, "p_bdpcm": 0.0} | (tu_kw or {})))
        irecs = None
    d = dict(cus=cus, pus=pus, ndmvr=ndmvr, tus=tus, coefs=coefs)
    p = A.Picture(); p.dstSlot = dst_slot; p.flags = 0
    if irecs is not None:
        d["intraTus"] = irecs; p.intraTus = irecs.ctypes.data; p.numIntraTus = len(irecs)
    if given is not None:                                       # pre-reconstructed samples (an intra picture's predictions stand in here)
        d["given"] = given
        for c in range(3): p.given[c] = given[c].ctypes.data
    p.pus = pus.ctypes.data; p.numPus = len(pus); p.numDmvr = ndmvr + 1
    p.tus = tus.ctypes.data; p.numTus = len(tus); p.coefs = coefs.ctypes.data; p.numCoefs = len(coefs)
    if deblock:
        qp = rng.integers(22, 45, size=len(cus))
        d["lfV"], d["lfH"] = gen_lf_grid(rng, cus, W, H, bit_depth, cu_intra=np.zeros(len(cus), bool) if cu_intra is None else np.ones(len(cus), bool) if cu_intra is True else cu_intra, cu_qp=qp)
        d["lfSlices"] = np.zeros(1, LFSLICE_DTYPE)
        p.flags |= A.PIC_DEBLOCK; p.lfV = d["lfV"].ctypes.data; p.lfH = d["lfH"].ctypes.data
        p.lfSlices = d["lfSlices"].ctypes.data; p.numLfSlices = 1
    if sao:
        d["sao"] = gen_sao(rng, W, H, ctu, bit_depth, p_on=sao_p)
        p.flags |= A.PIC_SAO; p.sao = d["sao"].ctypes.data
    if alf:
        d["alf"] = gen_alf(rng, W, H, ctu, bit_depth, **(alf_kw or {}))
        d["alfTabs"] = A.make_alf_tables(d["alf"])
        p.flags |= A.PIC_ALF; p.alf = d["alf"]["ctus"].ctypes.data; p.alfTabs = C.addressof(d["alfTabs"])
    if wp:   # explicit weighted prediction: such pictures carry no BDOF / DMVR PUs (pass pu_kw=dict(p_dmvr=0, p_bdof=0))
        d["wpRaw"], d["wp"] = gen_wp(rng, bit_depth, pus)
        p.wp = d["wp"].ctypes.data; p.numWp = len(d["wp"])
    if lmcs:
        d["lmcs"] = gen_lmcs(rng, bit_depth, cus, W, H, ctu, chroma_adj=lmcs_chroma)
        p.flags |= A.PIC_LMCS; p.lmcs = C.addressof(d["lmcs"]["struct"])
    d["struct"] = p
    return d


# ---- a whole picture as a flat dict of arrays (golden fixtures): save_picture(d) -> {name: ndarray}, load_picture(z) -> the dict of gen_picture
def save_picture(d):
    out = dict(pus=d["pus"], ndmvr=np.int64(d["ndmvr"]), tus=d["tus"], coefs=d["coefs"], dstSlot=np.int64(d["struct"].dstSlot))
    for k in ("lfV", "lfH", "lfSlices", "sao", "wp", "wpRaw"):
        if k in d: out[k] = d[k]
    if "alf" in d:
        a = d["alf"]
        out.update(alf_ctus=a["ctus"], alf_lumaCoeff=a["lumaCoeff"][16:], alf_lumaClip=a["lumaClip"][16:], alf_chromaCoeff=a["chromaCoeff"],
                   alf_chromaClip=a["chromaClip"], alf_cc0=a["cc"][0], alf_cc1=a["cc"][1])
    if "lmcs" in d:
        L = d["lmcs"]["struct"]
        out.update(lmcs_scalars=np.array([L.chromaAdj, L.minBinIdx, L.maxBinIdx, L.orgCW], np.int32), lmcs_reshapePivot=np.array(list(L.reshapePivot), np.int16),
                   lmcs_inputPivot=np.array(list(L.inputPivot), np.int16), lmcs_fwdScaleCoef=np.array(list(L.fwdScaleCoef), np.int16),
                   lmcs_chromaAdjHelpLUT=np.array(list(L.chromaAdjHelpLUT), np.int32), lmcs_invLUT=d["lmcs"]["invLUT"], lmcs_vpdus=d["lmcs"]["vpdus"])
    return out


def load_picture(z, bit_depth):
    """z: mapping from save_picture (e.g. an opened .npz)."""
    fixed_sets = (_fixed_sets(), np.full((16, 4, 25, 13), 1 << bit_depth, np.int16))
    from . import abi as A
    import ctypes as C
    d = dict(pus=np.ascontiguousarray(z["pus"]), ndmvr=int(z["ndmvr"]), tus=np.ascontiguousarray(z["tus"]), coefs=np.ascontiguousarray(z["coefs"]))
    p = A.Picture(); p.dstSlot = int(z["dstSlot"]); p.flags = 0
    p.pus = d["pus"].ctypes.data; p.numPus = len(d["pus"]); p.numDmvr = d["ndmvr"] + 1
    p.tus = d["tus"].ctypes.data; p.numTus = len(d["tus"]); p.coefs = d["coefs"].ctypes.data; p.numCoefs = len(d["coefs"])
    if "lfV" in z:
        for k in ("lfV", "lfH", "lfSlices"): d[k] = np.ascontiguousarray(z[k])
        p.flags |= A.PIC_DEBLOCK; p.lfV = d["lfV"].ctypes.data; p.lfH = d["lfH"].ctypes.data; p.lfSlices = d["lfSlices"].ctypes.data; p.numLfSlices = len(d["lfSlices"])
    if "sao" in z:
        d["sao"] = np.ascontiguousarray(z["sao"]); p.flags |= A.PIC_SAO; p.sao = d["sao"].ctypes.data
    if "alf_ctus" in z:
        d["alf"] = dict(ctus=np.ascontiguousarray(z["alf_ctus"]), lumaCoeff=np.ascontiguousarray(np.concatenate([fixed_sets[0], z["alf_lumaCoeff"]])),
                        lumaClip=np.ascontiguousarray(np.concatenate([fixed_sets[1], z["alf_lumaClip"]])), chromaCoeff=np.ascontiguousarray(z["alf_chromaCoeff"]),
                        chromaClip=np.ascontiguousarray(z["alf_chromaClip"]), cc=[np.ascontiguousarray(z["alf_cc0"]), np.ascontiguousarray(z["alf_cc1"])])
        d["alfTabs"] = A.make_alf_tables(d["alf"])
        p.flags |= A.PIC_ALF; p.alf = d["alf"]["ctus"].ctypes.data; p.alfTabs = C.addressof(d["alfTabs"])
    if "wp" in z:
        d["wp"] = np.ascontiguousarray(z["wp"]); d["wpRaw"] = np.ascontiguousarray(z["wpRaw"]); p.wp = d["wp"].ctypes.data; p.numWp = len(d["wp"])
    if "lmcs_scalars" in z:
        L = A.Lmcs(); sc = z["lmcs_scalars"]; L.chromaAdj, L.minBinIdx, L.maxBinIdx, L.orgCW = [int(v) for v in sc]
        for i in range(17): L.reshapePivot[i] = int(z["lmcs_reshapePivot"][i]); L.inputPivot[i] = int(z["lmcs_inputPivot"][i])
        for i in range(16): L.fwdScaleCoef[i] = int(z["lmcs_fwdScaleCoef"][i]); L.chromaAdjHelpLUT[i] = int(z["lmcs_chromaAdjHelpLUT"][i])
        lut = np.ascontiguousarray(z["lmcs_invLUT"]); vp = np.ascontiguousarray(z["lmcs_vpdus"])
        L.invLUT = lut.ctypes.data; L.vpdus = vp.ctypes.data
        d["lmcs"] = dict(struct=L, invLUT=lut, vpdus=vp)
        p.flags |= A.PIC_LMCS; p.lmcs = C.addressof(L)
    d["struct"] = p
    return d


# ---------------------------------------------------------------------------------------------------------------- film grain
def gen_fgc_sei(rng, model_id=0, present=(1, 1, 1), max_intervals=4, max_scale=200):
    """Film grain characteristics SEI parameters in the flat int layout oracle/ref_shim.cpp:ref_film_grain reads: modelId, log2ScaleFactor, then
    per component present, numModelValues, numIntervals and per interval lower, upper, 6 model values (vvdecSEIFilmGrainCharacteristics, sei.h:208).
    Frequency-filtering model (0): values = scale, h cutoff, v cutoff (2..14); auto-regressive model (1): scale, AR coefficients."""
    out = [model_id, int(rng.integers(2, 6))]
    for c in range(3):
        if not present[c]: out += [0, 0, 0]; continue
        n = int(rng.integers(1, max_intervals + 1))
        bounds = np.sort(rng.choice(np.arange(1, 255), size=2 * n, replace=False))
        nv = 3 if model_id == 0 else 6
        out += [1, nv, n]
        for i in range(n):
            if model_id == 0: vals = [int(rng.integers(20, max_scale)), int(rng.integers(2, 15)), int(rng.integers(2, 15)), 0, 0, 0]
            else: vals = [int(rng.integers(20, max_scale)), int(rng.integers(-60, 60)), int(rng.integers(-30, 30)), int(rng.integers(-30, 30)), 1 << out[1], int(rng.integers(-20, 20))]
            out += [int(bounds[2 * i]), int(bounds[2 * i + 1])] + vals
    return np.array(out, np.int32)


def gen_film_grain_tables(rng, H):
    """Random tables in the shape FilmGrainImpl holds them (no SEI / firmware involved): for device-vs-oracle tests on the GPU box."""
    pattern = rng.integers(-127, 128, size=(2, 8, 64, 64)).astype(np.int8)
    sLUT = rng.integers(0, 256, size=(3, 256)).astype(np.uint8)
    pLUT = (rng.integers(0, 8, size=(3, 256)) << 4).astype(np.uint8)
    seeds = rng.integers(0, 1 << 32, size=(H + 15) // 16, dtype=np.uint64).astype(np.uint32)
    return pattern, sLUT, pLUT, seeds


# ---------------------------------------------------------------------------------------------------------------- intra layouts
REF_INTRA_CU_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("w", "<u2"), ("h", "<u2"), ("dirL", "u1"), ("dirC", "u1"), ("multiRefIdx", "u1"), ("bdpcm", "u1"),
                               ("bdpcmC", "u1"), ("rsv", "u1", 3)])


def gen_intra_layout(rng, W, H, ctu=128, min_size=8, max_size=64, p_split=0.75):
    """CU rectangles (luma samples) of a picture in decoding order: CTUs in raster order, inside a CTU a random quad / binary tree in z-order
    (every CU at most max_size wide and high: one TU per CU)."""
    out = []

    def rec(x, y, w, h):
        if x >= W or y >= H: return
        must = w > max_size or h > max_size or x + w > W or y + h > H
        can_q = w == h and w // 2 >= min_size
        can_v, can_h = w // 2 >= min_size, h // 2 >= min_size
        if must or ((can_q or can_v or can_h) and rng.random() < p_split):
            opts = ([0] if can_q else []) + ([] if must and (w > max_size and h > max_size) else ([1] if can_v else []) + ([2] if can_h else []))
            if not opts: opts = [0]
            k = opts[int(rng.integers(len(opts)))]
            if k == 0:
                for dy in (0, h // 2):
                    for dx in (0, w // 2): rec(x + dx, y + dy, w // 2, h // 2)
            elif k == 1: rec(x, y, w // 2, h); rec(x + w // 2, y, w // 2, h)
            else: rec(x, y, w, h // 2); rec(x, y + h // 2, w, h // 2)
        else:
            out.append((x, y, w, h))

    for cy in range(0, H, ctu):
        for cx in range(0, W, ctu): rec(cx, cy, ctu, ctu)
    return out


_INTRA_ANG = [0, 1, 2, 3, 4, 6, 8, 10, 12, 14, 16, 18, 20, 23, 26, 29, 32, 35, 39, 45, 51, 57, 64, 73, 86, 102, 128, 171, 256, 341, 512, 1024]
_INTRA_THR = [24, 24, 24, 14, 2, 0, 0, 0]


def intra_wide_angle(w, h, mode):
    """IntraPrediction::getWideAngle (IntraPrediction.cpp:443)."""
    if 1 < mode <= 66:
        shift = [0, 6, 10, 12, 14, 15][abs(int(np.log2(w)) - int(np.log2(h)))]
        if w > h and mode < 2 + shift: return mode + 65
        if h > w and mode > 66 - shift: return mode - 65
    return mode


def intra_filter_ref(w, h, mode, mrl, bdpcm):
    """IntraPrediction::useFilteredIntraRefSamples (:1301) for a luma block."""
    if mrl or bdpcm or mode == 1: return False
    if mode == 0: return w * h > 32
    pm = intra_wide_angle(w, h, mode)
    diff = min(abs(pm - 18), abs(pm - 50))
    ang = _INTRA_ANG[abs(pm - 50 if pm >= 34 else -(pm - 18))]
    return diff > _INTRA_THR[(int(np.log2(w)) + int(np.log2(h))) >> 1] and (ang & 31) == 0


def isp_regions(w, h, split):
    """Prediction regions (dx, dy, rw, rh) of an ISP CU and the width of its transform units (CU::getISPSplitDim UnitTools.cpp:360, isPredRegDiffFromTB):
    split 1 = horizontal (regions stacked), 2 = vertical; vertical sub-partitions narrower than 4 share a 4-wide region."""
    sd, nd = (h, w) if split == 1 else (w, h)
    part = max(sd >> 2, 16 // nd if nd < 16 else 1)
    if split == 1: return [(0, k * part, w, part) for k in range(h // part)], w
    rw = max(part, 4)
    return [(k * rw, 0, rw, h) for k in range(w // rw)], part


def gen_intra_records(rng, layout, W, H, modes=None, p_mrl=0.15, p_bdpcm=0.08, p_resi=0.0, upto=None, only=None, p_mip=0.15, colloc=0, p_lm=0.0, ciip=None, p_isp=0.0, ctu=128):
    """b200_intra_tu records (Y, Cb, Cr per CU, decoding order) for a single-tree all-intra layout of gen_intra_layout: random modes, MRL on some luma
    blocks (never on the first row of a CTU of size `ctu`, the layout's), BDPCM prediction on some, availability as xFillReferenceSamples derives it
    from the decoding order (pinned against the reference's own analysis through the glue flattener by tests/test_intra_oracle_vs_ref.py).  Luma blocks
    whose chroma would be narrower than 4 or smaller than 16 samples are luma-only (local dual tree; their chroma is not generated)."""
    A = abi
    owner = np.full(((H + 3) // 4, (W + 3) // 4), 1 << 30, np.int64)
    for i, (x, y, w, h) in enumerate(layout): owner[y // 4:(y + h) // 4, x // 4:(x + w) // 4] = i
    recs = []
    chroma_modes = [0, 1, 18, 50, 2, 34, 66, -1, -1, -1, 23, 45, 61]
    for i, (x, y, w, h) in enumerate(layout if upto is None else layout[:upto + 1]):
        mip = 0
        if modes is not None and i in modes:
            m = modes[i]; dirL, dirC, mrl, bdpcm = m[:4]; mip = m[4] if len(m) > 4 else 0
        else:
            dirL, mrl, bdpcm = int(rng.integers(0, 67)), 0, 0
            if rng.random() < p_mrl and y % ctu: mrl, dirL = int(rng.integers(1, 3)), int(rng.integers(1, 67))
            elif rng.random() < p_bdpcm and w <= 32 and h <= 32: bdpcm = int(rng.integers(1, 3))
            elif rng.random() < p_mip:                                   # matrix intra prediction: dirL is the MIP mode index of the size class
                n_modes = 16 if (w, h) == (4, 4) else 8 if (w == 4 or h == 4 or (w, h) == (8, 8)) else 6
                dirL, mip = int(rng.integers(0, n_modes)), 1 | (int(rng.integers(0, 2)) << 1)
            dirC = chroma_modes[int(rng.integers(len(chroma_modes)))]
            if rng.random() < p_lm: dirC = int(rng.integers(67, 70))
        if dirC < 0 or dirC == 70: dirC = 0 if mip else dirL            # DM (a MIP luma CU counts as planar: PU::getCoLocatedIntraLumaMode)
        wc = ciip.get(i, 0) if ciip else 0                              # CIIP CU (inter): planar blocks blended with the inter prediction, weight wc
        if wc: dirL, dirC, mrl, bdpcm, mip = 0, 0, 0, 0, 0
        lm = dirC in (67, 68, 69)                                       # LM_CHROMA_IDX, MDLM_L_IDX, MDLM_T_IDX
        if only is not None and not only[i]: continue                   # an inter CU of a mixed picture: a neighbour, not a block of the list
        def avail(ux, uy): return 0 <= ux < owner.shape[1] and 0 <= uy < owner.shape[0] and owner[uy, ux] < i
        tl = avail(x // 4 - 1, y // 4 - 1)
        na = 0
        while na < 2 * w // 4 and avail(x // 4 + na, y // 4 - 1): na += 1
        nl = 0
        while nl < 2 * h // 4 and avail(x // 4 - 1, y // 4 + nl): nl += 1
        luma_only = w < 8 or (w // 2) * (h // 2) < 16
        if wc: luma_only = (w // 2) <= 2
        isp = 0
        if p_isp and not (mip or mrl or bdpcm or wc) and w * h > 16 and rng.random() < p_isp: isp = int(rng.integers(1, 3))
        if isp:
            # intra sub-partitions: one record per prediction region, the CU-level neighbourhood in each (include/vvdec_b200.h, B200_INTRA_ISP)
            regions, tuw = isp_regions(w, h, isp)
            for k, (dx, dy, rw, rh) in enumerate(regions):
                r = np.zeros((), A.INTRA_TU_DTYPE)
                r["x"], r["y"], r["log2w"], r["log2h"], r["mode"] = x + dx, y + dy, int(np.log2(rw)), int(np.log2(rh)), dirL
                r["mip"] = isp | (k << 2) | (int(np.log2(len(regions))) << 4)
                mask = int(rng.integers(0, 1 << (rw // tuw))) if rng.random() < max(p_resi, 0.0) * 1.5 else 0
                r["ciip"] = mask
                r["flags"] = A.INTRA_ISP | (A.INTRA_AVAIL_TL if tl else 0) | (4 if mask else 0)
                r["numAbove"], r["numLeft"], r["lmLeft"], r["lmAbove"] = na, nl, int(avail(x // 4 - 1, y // 4)), int(avail(x // 4, y // 4 - 1))
                recs.append(r)
        for c in range(1 if luma_only else 3):
            if isp and c == 0: continue
            r = np.zeros((), A.INTRA_TU_DTYPE)
            r["ciip"] = wc
            sh = 1 if c else 0
            r["x"], r["y"], r["log2w"], r["log2h"], r["comp"] = x >> sh, y >> sh, int(np.log2(w >> sh)), int(np.log2(h >> sh)), c
            if c == 0 and mip: r["mode"], r["mip"] = A.INTRA_MIP, dirL | ((mip >> 1) << 7)
            elif c == 0: r["mode"] = (A.INTRA_BDPCM_HOR if bdpcm == 1 else A.INTRA_BDPCM_VER) if bdpcm else dirL
            else: r["mode"] = dirC + 3 if lm else dirC                # B200_INTRA_LM = 70 ...
            r["multiRefIdx"] = mrl if c == 0 else 0
            fl = A.INTRA_AVAIL_TL if tl else 0
            if c == 0 and not mip and intra_filter_ref(w, h, dirL, mrl, bdpcm): fl |= A.INTRA_FILTER_REF
            if rng.random() < p_resi: fl |= 4
            if c and lm:
                cw, chh = w >> 1, h >> 1
                if na: fl |= A.INTRA_LM_ABOVE
                if nl: fl |= A.INTRA_LM_LEFT
                if colloc: fl |= A.INTRA_LM_COLLOCATED
                r["lmAbove"] = cw // 2 if na else 0; r["lmLeft"] = chh // 2 if nl else 0
                if dirC == 69 and na: r["lmAbove"] = min(na, cw // 2 + min(cw // 2, chh // 2))
                if dirC == 68 and nl: r["lmLeft"] = min(nl, chh // 2 + min(chh // 2, cw // 2))
            r["flags"], r["numAbove"], r["numLeft"] = fl, na, nl
            recs.append(r)
    return np.array(recs, A.INTRA_TU_DTYPE)


# ---------------------------------------------------------------------------------------------------------------- designed intra sweep
def intra_sweep_blocks():
    """The blocks of the designed K6 sweep, as (comp, w, h, mode, multiRefIdx, mip): every luma shape 4x4 .. 64x64 with every mode 0..66, MRL 1 and 2 with
    every angular mode, BDPCM H / V up to 32x32 and every MIP mode of the size class, transposed and not; every chroma shape 4x4 .. 32x32 of Cb and Cr with
    every mode 0..66."""
    A = abi
    out = []
    sizes = (4, 8, 16, 32, 64)
    for w in sizes:
        for h in sizes:
            out += [(0, w, h, m, 0, 0) for m in range(67)]
            out += [(0, w, h, m, mrl, 0) for mrl in (1, 2) for m in range(2, 67)]
            if w <= 32 and h <= 32: out += [(0, w, h, A.INTRA_BDPCM_HOR, 0, 0), (0, w, h, A.INTRA_BDPCM_VER, 0, 0)]
            n_mip = 16 if (w, h) == (4, 4) else 8 if (w == 4 or h == 4 or (w, h) == (8, 8)) else 6
            out += [(0, w, h, A.INTRA_MIP, 0, k | (tr << 7)) for k in range(n_mip) for tr in (0, 1)]
    for c in (1, 2):
        out += [(c, w, h, m, 0, 0) for w in sizes[:4] for h in sizes[:4] for m in range(67)]
    return out


INTRA_SWEEP_AVAIL = ("full", "partial", "none")


def _sweep_slots(cx, cy, C, W, H, w, h, gap):
    """Positions of a w x h block grid inside the CTU (cx, cy, size C) of a W x H plane.  Every block keeps `gap` free columns left of it and `gap` free rows
    above it (its reference row / column, MRL lines included), and its above-right and below-left references (2w, 2h) end inside the CTU or the free band
    in front of the next CTU.  So no block's reference samples are another block's samples: every reference is noise, nothing depends on anything."""
    xs = [x for x in range(cx + gap, cx + C, w + gap) if x + w <= cx + C and x + 2 * w <= min(cx + C + gap, W)]
    ys = [y for y in range(cy + gap, cy + C, h + gap) if y + h <= cy + C and y + 2 * h <= min(cy + C + gap, H)]
    return [(x, y) for y in ys for x in xs]


def intra_sweep(ctu=128, ctus_w=32):
    """The designed sweep as one list: every block of intra_sweep_blocks() once per neighbourhood of INTRA_SWEEP_AVAIL (full: numAbove = 2w / unit,
    numLeft = 2h / unit and the corner; partial: above-right or below-left cut, no corner; none), placed on a grid of noise in CTU raster order with each
    CTU's records contiguous (luma, Cb, Cr).  Luma reference filtering as intra_filter_ref says; every record carries INTRA_ADD_RESI.
    Returns (W, H, records); the picture is ctus_w CTUs wide and has one empty CTU row at the bottom."""
    A = abi
    blocks = intra_sweep_blocks()
    groups = {}                                                   # (luma?, w, h) -> [(comp, mode, mrl, mip, avail)], Cb and Cr of a shape side by side
    for (c, w, h, mode, mrl, mip) in blocks:
        for av in INTRA_SWEEP_AVAIL: groups.setdefault((c == 0, w, h), []).append((c, mode, mrl, mip, av))
    W = ctus_w * ctu
    per_ctu = {}                                                  # CTU index -> records
    for luma in (True, False):
        C, gap, sh = (ctu, 4, 0) if luma else (ctu // 2, 2, 1)
        Wc = W >> sh
        k = 0                                                     # next CTU of this channel
        for (l, w, h), todo in groups.items():
            if l != luma: continue
            cr = None if luma else [b for b in todo if b[0] == 2]  # Cr blocks at the positions of the Cb blocks, in their own plane
            if not luma: todo = [b for b in todo if b[0] == 1]
            i = 0
            while i < len(todo):
                cx, cy = (k % ctus_w) * C, (k // ctus_w) * C
                slots = _sweep_slots(cx, cy, C, Wc, 1 << 30, w, h, gap)
                for (x, y) in slots:
                    if i >= len(todo): break
                    for b in ([todo[i]] if luma else [todo[i], cr[i]]):
                        per_ctu.setdefault(k, []).append((b[0], x, y, w, h) + b[1:])
                    i += 1
                k += 1
    n_ctu = max(per_ctu) + 1
    H = ((n_ctu + ctus_w - 1) // ctus_w + 1) * ctu
    recs = []
    for k in sorted(per_ctu):
        for j, (c, x, y, w, h, mode, mrl, mip, av) in enumerate(sorted(per_ctu[k], key=lambda r: r[0])):
            r = np.zeros((), A.INTRA_TU_DTYPE)
            unit = 2 if c else 4
            r["x"], r["y"], r["log2w"], r["log2h"], r["comp"], r["mode"], r["multiRefIdx"], r["mip"] = x, y, int(np.log2(w)), int(np.log2(h)), c, mode, mrl, mip
            fl = A.INTRA_ADD_RESI
            if av == "full": fl |= A.INTRA_AVAIL_TL; r["numAbove"], r["numLeft"] = 2 * w // unit, 2 * h // unit
            elif av == "partial":
                if j & 1: r["numAbove"], r["numLeft"] = w // unit, 2 * h // unit
                else: r["numAbove"], r["numLeft"] = 2 * w // unit, h // unit
            if c == 0 and mode <= 66 and intra_filter_ref(w, h, mode, mrl, 0): fl |= A.INTRA_FILTER_REF
            r["flags"] = fl
            recs.append(r)
    return W, H, np.array(recs, A.INTRA_TU_DTYPE)


def intra_record_key(r):
    """(comp, w, h, mode, multiRefIdx, mip) of a record: the block identity intra_sweep_blocks() lists."""
    return (int(r["comp"]), 1 << int(r["log2w"]), 1 << int(r["log2h"]), int(r["mode"]), int(r["multiRefIdx"]), int(r["mip"]))


# ---------------------------------------------------------------------------------------------------------------- designed CCLM sweep
# Chroma CCLM records (modes LM, MDLM_L, MDLM_T) over 4:2:0 planes, as named cases (tests/test_k6_*.py):
#   geometry_ctu{32,64,128}: every chroma shape the reference codes with every LM / MDLM neighbourhood, under each luma down-sampling filter (3-tap on
#     the first row of a CTU, 5-tap collocated, 6-tap), blocks without a left / above CU also at the picture's left / top edge; on noise.
#   targets_{8,10,12}bit: 8x8 blocks whose templates are written so that the four selected (luma, chroma) pairs reach each target of the parameter
#     derivation (CCLM_TARGETS) with both selections (two above + two left, four from one side), and 2-high blocks on the two-sample path.
#   chained: luma blocks earlier in the list write the templates (in the CTUs above and to the left) and the co-located luma of the CCLM blocks.
# Every block owns its footprint: the two chroma rows / columns in front of it and its 2w x 2h reference reach (the luma footprint is twice that).
# Footprints never overlap, so no block reads another block's output (except in the chained case, on purpose) or another block's designed samples.
CCLM_SHAPES = tuple((w, h) for w in (4, 8, 16, 32) for h in (2, 4, 8, 16, 32) if w * h >= 16)
CCLM_WEAK_ORDERS = tuple(sorted({tuple(sorted(set(r)).index(v) for v in r) for r in np.ndindex(4, 4, 4, 4)}))      # the 75 weak orderings of 4 samples
CCLM_TARGETS = (tuple(("tie",) + o for o in CCLM_WEAK_ORDERS) + (("diff0",), ("diffC0",)) + tuple(("normDiff", n, s) for n in range(16) for s in (1, -1))
                + (("clamp", 1), ("clamp", -1), ("clip0",), ("clipmax",), ("luma0",), ("lumamax",)))
CCLM_SWEEP_CASES = {
    "geometry_ctu32": ("geometry", 32, 10), "geometry_ctu64": ("geometry", 64, 8), "geometry_ctu128": ("geometry", 128, 12),
    "targets_8bit": ("targets", 128, 8), "targets_10bit": ("targets", 128, 10), "targets_12bit": ("targets", 128, 12),
    "chained": ("chained", 64, 10),
}


def cclm_picks(num, alone):
    """Template positions xGetLMParameters selects from `num` samples of one side: two, or four when the other side is absent (`alone`)."""
    start, step = num >> (2 + alone), max(1, num >> (1 + alone))
    return [start + k * step for k in range(min(num, (1 + alone) << 1))]


def cclm_neighbourhoods(w, h):
    """(mode, above, left, lmAbove, lmLeft, numAbove, numLeft) of every LM / MDLM neighbourhood of a w x h chroma block, consistent as the glue
    flattener derives them (flatten_intra.h:102-112): LM with each (above, left) pair; MDLM_T with lmAbove at w/2, in between and at its largest
    (w/2 + min(w/2, h/2) units, the above-right units available), and without an above CU; MDLM_L likewise."""
    A = abi
    out = [(A.INTRA_LM, a, l, w // 2 * a, h // 2 * l, w * a, h * l) for a in (1, 0) for l in (1, 0)]
    for mode, n, m in ((A.INTRA_MDLM_T, w, h), (A.INTRA_MDLM_L, h, w)):
        lo, hi = n // 2, n // 2 + min(n // 2, m // 2)
        for v in sorted({lo, (lo + hi) // 2, hi}) + [0]:
            side = (v, n // 2 + (v - lo if v else 0)) if v else (0, 0)            # (lm units, available units of 2n): the units beyond n are above-right / below-left
            other = (m // 2, m)
            if mode == A.INTRA_MDLM_T: out.append((mode, int(v > 0), 1, side[0], other[0], side[1], other[1]))
            else: out.append((mode, 1, int(v > 0), other[0], side[0], other[1], side[1]))
    return out


def _cclm_record(x, y, w, h, comp, nb, colloc):
    mode, above, left, lmA, lmL, numA, numL = nb
    r = np.zeros((), abi.INTRA_TU_DTYPE)
    r["x"], r["y"], r["log2w"], r["log2h"], r["comp"], r["mode"] = x, y, int(np.log2(w)), int(np.log2(h)), comp, mode
    fl = abi.INTRA_ADD_RESI | (abi.INTRA_AVAIL_TL if above and left else 0) | (abi.INTRA_LM_ABOVE if above else 0) | (abi.INTRA_LM_LEFT if left else 0)
    r["flags"] = fl | (abi.INTRA_LM_COLLOCATED if colloc else 0)
    r["lmAbove"], r["lmLeft"], r["numAbove"], r["numLeft"] = lmA, lmL, numA, numL
    return r


def _cclm_pack(blocks, C, ctus_w, gap=2):
    """Positions of blocks [(w, h, where)] in CTU raster order (size C, ctus_w CTUs a row): the first position on the `gap`-sample grid inside a CTU
    where the block's footprint (its `gap` reference rows / columns in front of it, its 2w x 2h reach) is free.  where: "any" (the first row of a CTU
    only where nothing else is free); "inner" (never the first row of a CTU: blocks with MRL); "first_row" (y on the first row of a CTU below the first); "left_edge" (x = 0); "top_edge" (y = 0).
    CCLM packs chroma blocks with gap 2; the regular intra sweep packs luma with gap 4 (MRL 2 reads the third row / column in front of a block)."""
    Wc = C * ctus_w
    occ = np.zeros((C * 128, Wc), bool)
    cursor, out = {}, [None] * len(blocks)
    for i in sorted(range(len(blocks)), key=lambda i: blocks[i][2] not in ("top_edge", "left_edge")):     # the edges first
        w, h, where = blocks[i]
        k = cursor.get((w, h, where), ctus_w if where == "first_row" else 0)
        while True:
            cx, cy = (k % ctus_w) * C, (k // ctus_w) * C
            xs = [x for x in range(cx, cx + C - w + 1, gap) if x >= gap]
            ys = [y for y in list(range(cy + gap, cy + C - h + 1, gap)) + [cy] if y >= gap]    # the first row of a CTU last: only a block as high as the CTU sits there
            slots = [(x, y) for y in ys for x in xs]
            cands = {"any": slots, "inner": [(x, y) for (x, y) in slots if y != cy], "first_row": [(x, cy) for x in xs], "left_edge": [(0, y) for y in ys] if cx == 0 else [],
                     "top_edge": [(x, 0) for x in xs] if cy == 0 else []}[where]
            cands = [(x, y) for (x, y) in cands if x + 2 * w <= Wc]
            if cands:                                                # the footprint sums of all candidates at once, from an integral image of the CTU's window
                X, Y = np.array(cands).T
                wx, wy = max(0, cx - gap), max(0, cy - gap)
                win = occ[wy:cy + C + 2 * h, wx:cx + C + 2 * w]
                ii = np.zeros((win.shape[0] + 1, win.shape[1] + 1), np.int32)
                ii[1:, 1:] = win.cumsum(0).cumsum(1)
                y0, y1, x0, x1 = np.maximum(0, Y - gap) - wy, Y + 2 * h - wy, np.maximum(0, X - gap) - wx, X + 2 * w - wx
                free = np.flatnonzero(ii[y1, x1] - ii[y0, x1] - ii[y1, x0] + ii[y0, x0] == 0)
                if len(free): hit = cands[free[0]]; break
            k += 1
            assert where != "top_edge" or k < ctus_w, "the top edge is full"
        cursor[(w, h, where)] = k
        x, y = hit
        occ[max(0, y - gap):y + 2 * h, max(0, x - gap):x + 2 * w] = True
        out[i] = hit
    return out


def cclm_paint(planes, x, y, w, h, rec, sel_l, sel_c, bd):
    """Writes the templates of the CCLM record `rec` at chroma (x, y) so that the luma down-sampled at the selected positions (above ones first, as
    xGetLMParameters takes them) is sel_l and the chroma there is sel_c (Cb; Cr gets pmax - sel_c), and the block's luma a ramp from 0 to pmax.  Luma
    is written as constant cells: every tap of a selected position lies in that position's cell where selected positions are at least two apart."""
    pmax = (1 << bd) - 1
    Y, Cb, Cr = planes
    mode, fl = int(rec["mode"]), int(rec["flags"])
    above, left = bool(fl & abi.INTRA_LM_ABOVE), bool(fl & abi.INTRA_LM_LEFT)
    top_n = 2 * int(rec["lmAbove"]) if mode == abi.INTRA_MDLM_T else w if mode == abi.INTRA_LM and above else 0
    left_n = 2 * int(rec["lmLeft"]) if mode == abi.INTRA_MDLM_L else h if mode == abi.INTRA_LM and left else 0
    pa = cclm_picks(top_n, int(not left_n)) if top_n else []
    pl = cclm_picks(left_n, int(not top_n)) if left_n else []
    assert len(pa) + len(pl) == len(sel_l)

    def cell(picks, vals, i):                                       # the value of the first selected position at or after template position i
        return next((v for p, v in zip(picks, vals) if p >= i), vals[-1])
    lx, ly = 2 * x, 2 * y
    for c in range(lx - 1, lx + 2 * top_n) if pa else ():            # rows above: position i reads columns 2i - 1 .. 2i + 1
        Y[ly - 3:ly, c] = cell(pa, sel_l[:len(pa)], (c - lx) // 2)
    for r in range(ly - 1, ly + 2 * left_n) if pl else ():           # columns left: position j reads rows 2j - 1 .. 2j + 1
        Y[r, lx - 3:lx - (1 if r < ly else 0)] = cell(pl, sel_l[len(pa):], (r - ly) // 2)
    ramp = np.clip(np.round((np.arange(2 * w) - w / 2) * pmax / w), 0, pmax)
    Y[ly:ly + 2 * h, lx:lx + 2 * w] = ramp[None, :]
    for p, v in zip(pa, sel_c[:len(pa)]): Cb[y - 1, x + p], Cr[y - 1, x + p] = v, pmax - v
    for p, v in zip(pl, sel_c[len(pa):]): Cb[y + p, x - 1], Cr[y + p, x - 1] = v, pmax - v


def cclm_target_values(t, bd, n=4):
    """(sel_l, sel_c): template values that reach target t (a CCLM_TARGETS entry; the clip and luma targets ride on the clamped slopes) with n
    selected samples (4, or 2 for the two-sample path, where t = ("tie2", order))."""
    u, mid = 1 << (bd - 8), 1 << (bd - 1)
    if t[0] == "tie2": return [mid - 40 * u + 40 * u * t[1], mid], [mid - 30 * u, mid + 50 * u]
    if t[0] == "tie": return [mid - 60 * u + 40 * u * r for r in t[1:]], [mid - 60 * u, mid + 20 * u, mid - 20 * u, mid + 60 * u]
    m, c = mid - 8 * u, mid + 3 * u
    if t[0] == "diff0": return [m] * 4, [c - 30, c + 10, c - 10, c + 30]
    if t[0] == "diffC0": return [m, m + 80 * u, m, m + 80 * u], [c] * 4
    if t[0] == "normDiff": d, dc = 16 + t[1], 20 * t[2]
    else: d, dc = 2, 100 * t[1]                                       # "clamp": diff 2, |diffC| 100: shift = 3 + 1 - 7 < 1
    return [m, m + d, m, m + d], [c, c + dc, c, c + dc]


def _cclm_geometry_blocks(C):
    """(w, h, nb, colloc, where) of a geometry case: each neighbourhood of each shape that fits a chroma CTU of size C under each filter, and the
    neighbourhoods without a left (above) CU once more at the picture's left (top) edge."""
    out = []
    for (w, h) in CCLM_SHAPES:
        if w > C or h > C: continue
        nbs = cclm_neighbourhoods(w, h)
        for k, nb in enumerate(nbs):
            out += [(w, h, nb, 0, "any"), (w, h, nb, 1, "any")]
            if nb[1]: out.append((w, h, nb, k & 1, "first_row"))
        out.append((w, h, nbs[1], 0, "left_edge"))                 # LM above only: m = 0 at i = 0
        out.append((w, h, nbs[2], 1, "top_edge"))                  # LM left only, collocated: up = 0 at j = 0
    return out


def _cclm_target_blocks(bd):
    """(w, h, nb, colloc, where, target, sel_l, sel_c) of a targets case: every target with two above + two left (LM), four above (LM above only /
    MDLM_T) and four left (LM left only / MDLM_L), on 8x8 blocks; the three orderings of the two-sample path on 8x2, 16x2 and 32x2 (LM left only)."""
    out = []
    nbs = cclm_neighbourhoods(8, 8)
    both, a_only, l_only = nbs[0], nbs[1], nbs[2]
    mdlm_t = [nb for nb in nbs if nb[0] == abi.INTRA_MDLM_T][2]        # lmAbove at its largest
    mdlm_l = [nb for nb in nbs if nb[0] == abi.INTRA_MDLM_L][2]
    for k, t in enumerate(CCLM_TARGETS):
        if t[0] in ("clip0", "clipmax", "luma0", "lumamax"): continue
        sel_l, sel_c = cclm_target_values(t, bd)
        for nb in (both, (a_only, mdlm_t)[k & 1], (l_only, mdlm_l)[k & 1]): out.append((8, 8, nb, k & 1, "any", t, sel_l, sel_c))
    for w in (8, 16, 32):
        for o in range(3):
            sel_l, sel_c = cclm_target_values(("tie2", o), bd)
            out.append((w, 2, cclm_neighbourhoods(w, 2)[2], 0, "any", ("tie2", o), sel_l, sel_c))
    return out


def _cclm_chained(ctu, bd, rng):
    """CCLM blocks at the top-left corner of the CTUs of the second CTU row, each after the luma blocks that write its templates: a 32x8 block in the
    CTU above (the above template), an 8x8 block in the CTU above-left (the corner), an 8x32 block in the CTU to the left (the left template) and the
    co-located block; planar luma (a flat DC template would make the slope 0) over noise, so it differs from the noise the planes start with.  The
    co-located block reads no neighbour, so it does not wait for the template blocks: only the CCLM block's own wait orders it after them."""
    A = abi
    n_ctu = 5
    W, H = (n_ctu + 1) * ctu, 3 * ctu
    luma, chroma = [], []
    nbs = cclm_neighbourhoods(8, 8)
    modes = [nbs[0], [nb for nb in nbs if nb[0] == A.INTRA_MDLM_T][2], [nb for nb in nbs if nb[0] == A.INTRA_MDLM_L][2], nbs[0], nbs[0]]
    for k in range(n_ctu):
        X = (k + 1) * ctu
        for (lx, ly, w, h) in ((X - 8, ctu - 8, 8, 8), (X, ctu - 8, 32, 8), (X - 8, ctu, 8, 32), (X, ctu, 16, 16)):
            r = np.zeros((), A.INTRA_TU_DTYPE)
            r["x"], r["y"], r["log2w"], r["log2h"], r["mode"] = lx, ly, int(np.log2(w)), int(np.log2(h)), 0
            if ly < ctu or lx < X:                                     # the template blocks; the co-located block has no neighbourhood of its own
                r["numAbove"], r["numLeft"] = 2 * w // 4, 2 * h // 4
                r["flags"] = A.INTRA_AVAIL_TL | (A.INTRA_FILTER_REF if intra_filter_ref(w, h, 0, 0, 0) else 0)
            r["flags"] |= A.INTRA_ADD_RESI
            luma.append(r)
        for comp in (1, 2): chroma.append(_cclm_record(X // 2, ctu // 2, 8, 8, comp, modes[k], k & 1))
    recs = np.array(luma + chroma, A.INTRA_TU_DTYPE)
    key = ((recs["y"].astype(int) << (recs["comp"] > 0)) // ctu) * (W // ctu) + ((recs["x"].astype(int) << (recs["comp"] > 0)) // ctu)
    return W, H, recs[np.argsort(key, kind="stable")], ["chained"] * len(recs)


_cclm_sweep_cache = {}


def cclm_sweep(name):
    """One case of the designed CCLM sweep (CCLM_SWEEP_CASES) as a dict: geometry (g, W, H, bd, ctu), noise planes with the designed templates
    written in (planes), the residual planes (resi), the records in CTU order (recs, Cb and Cr of each block) and per record what it was built for
    (tags: the neighbourhood / filter / edge of a geometry block, the target of a targets block, Cr's with the chroma slope negated)."""
    if name in _cclm_sweep_cache: return _cclm_sweep_cache[name]
    kind, ctu, bd = CCLM_SWEEP_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    C = ctu // 2
    if kind == "chained":
        W, H, recs, tags = _cclm_chained(ctu, bd, rng)
        planes = noise_planes(rng, W, H, bd)
    else:
        blocks = _cclm_geometry_blocks(C) if kind == "geometry" else _cclm_target_blocks(bd)
        ctus_w = max(8, 1024 // C)
        pos = _cclm_pack([(b[0], b[1], b[4]) for b in blocks], C, ctus_w)
        W = ctus_w * ctu
        H = ((max(y + 2 * b[1] for (x, y), b in zip(pos, blocks)) + C - 1) // C + 1) * ctu
        planes = noise_planes(rng, W, H, bd)
        per = []
        for (x, y), b in zip(pos, blocks):
            w, h, nb, colloc, where = b[:5]
            tag = ("geometry", nb, colloc, where) if kind == "geometry" else b[5]
            rs = [_cclm_record(x, y, w, h, comp, nb, colloc) for comp in (1, 2)]
            if kind == "targets": cclm_paint(planes, x, y, w, h, rs[0], b[6], b[7], bd)
            neg = (tag[0], tag[1], -tag[2]) if tag[0] == "normDiff" else (tag[0], -tag[1]) if tag[0] == "clamp" else tag
            per += [(rs[0], tag), (rs[1], neg)]
        key = [((int(r["y"]) * 2) // ctu) * (W // ctu) + (int(r["x"]) * 2) // ctu for r, _ in per]
        order = np.argsort(key, kind="stable")
        recs = np.array([per[i][0] for i in order], abi.INTRA_TU_DTYPE)
        tags = [per[i][1] for i in order]
    g = abi.make_geom(W, H, bd, ctu=ctu)
    resi = [rng.integers(-64, 65, size=p.shape).astype(np.int16) for p in planes]
    case = dict(name=name, g=g, W=W, H=H, bd=bd, ctu=ctu, planes=planes, resi=resi, recs=recs, tags=tags)
    _cclm_sweep_cache[name] = case
    return case


# ---------------------------------------------------------------------------------------------------------------- designed regular intra sweep
# Regular intra records (planar, DC, angular, MRL, PDPC, BDPCM, MIP) on designed reference samples, as named cases (tests/test_k6_*.py):
#   regular_targets_{8,10,12}bit: each block's reference rows and columns are written so that a clip site of the prediction sees values below 0 and above
#     pmax (INTRA_TARGETS: the cubic interpolation of fractional luma angles with MRL 0, 1 and 2, PDPC of modes 18 and 50, the reduced MIP prediction
#     of each size class, transposed and not), substitution takes the mid value (no neighbour) or pads from one available unit at 0 or pmax, BDPCM
#     copies references at 0 and pmax; the residual is large enough that pred + resi crosses 0 and pmax in every component.
#   regular_flat_{8,12}bit: every reference sample (MRL lines included) of a block holds one value v in {0, 1, mid, pmax - 1, pmax}, with full and partial
#     neighbourhoods: planar, DC, every angular mode, MRL 1 and 2 (every third angular mode), BDPCM on every shape.  Every predicted sample is v (MIP is left out: its output on
#     flat input is not v).
#   regular_geometry_ctu{32,64}: the targets blocks of every shape that fits the CTU (8 and 12 bit), blocks without a neighbour also at the picture's
#     top and left edges; regular_stride_odd_12bit: the same at CTU 128 on planes with odd, padded strides (the one-CTA-per-block path);
#     regular_yuv400_10bit: luma only (CTU 64).
#   regular_chained: consumer blocks whose last above-right unit, last below-left unit, corner and MRL line 2 are written by earlier producer blocks, in the
#     CTU above, the CTU to the left, the CTU above-right and the CTU itself, at 12 bit with producers at 0 and pmax.
# Every block owns its footprint: its reference rows / columns (4 luma, 2 chroma: MRL lines included), its 2w / 2h reach and its corner.  Footprints
# never overlap (except in the chained case), so no block reads another block's samples.
INTRA_LUMA_SHAPES = tuple((w, h) for w in (4, 8, 16, 32, 64) for h in (4, 8, 16, 32, 64))
INTRA_CHROMA_SHAPES = tuple((w, h) for w in (4, 8, 16, 32) for h in (4, 8, 16, 32))
INTRA_TARGETS = ("cubic_lo", "cubic_hi", "pdpc_lo", "pdpc_hi", "mip_lo", "mip_hi", "subst_mid", "pad_0", "pad_max", "reco_lo", "reco_hi", "bdpcm")
INTRA_SWEEP_CASES = {
    "regular_targets_8bit": ("targets", 128, 8, None, True), "regular_targets_10bit": ("targets", 128, 10, None, True), "regular_targets_12bit": ("targets", 128, 12, None, True),
    "regular_flat_8bit": ("flat", 128, 8, None, True), "regular_flat_12bit": ("flat", 128, 12, None, True),
    "regular_geometry_ctu32": ("targets", 32, 8, None, True), "regular_geometry_ctu64": ("targets", 64, 12, None, True),
    "regular_stride_odd_12bit": ("targets", 128, 12, 7, True), "regular_yuv400_10bit": ("targets", 64, 10, None, False),
    "regular_chained": ("chained", 64, 12, None, True),
}


def intra_mip_modes(w, h):
    """Number of MIP modes of a w x h luma block's size class (getMipSizeId: 4x4; 4xN, Nx4 and 8x8; the rest)."""
    return 16 if (w, h) == (4, 4) else 8 if (w == 4 or h == 4 or (w, h) == (8, 8)) else 6


def intra_cubic_modes(w, h, mrl):
    """Up to three angular modes of a w x h luma block that interpolate a fractional angle with the cubic filter: with MRL every fractional angle
    does; without it only angles close enough to horizontal / vertical for the block size (intra_filter_ref's threshold).  Spread over the range."""
    out = []
    for m in range(2, 67):
        pm = intra_wide_angle(w, h, m)
        a = _INTRA_ANG[abs(pm - 50 if pm >= 34 else -(pm - 18))]
        diff = min(abs(pm - 18), abs(pm - 50))
        if a & 31 and (mrl or diff <= _INTRA_THR[(int(np.log2(w)) + int(np.log2(h))) >> 1]): out.append(m)
    return [out[i] for i in sorted({0, len(out) // 2, len(out) - 1})] if out else []


def _intra_pattern(kind, bd, v=0):
    """pattern(k, n, left): the value of reference sample k of a block whose side is n samples long (k = 0: the corner, k >= 1: the k-th sample of the
    row above, or of the column to the left, k < 0: the MRL corner)."""
    pmax, mid = (1 << bd) - 1, 1 << (bd - 1)
    return {"cubic": lambda k, n, l: pmax if (k // 2) % 2 else 0,                 # 0 0 pmax pmax 0 0 ...: 4-tap windows across a step overshoot
            "pdpc": lambda k, n, l: mid if k <= 0 else pmax if k % 2 else 0,      # corner mid, sides pmax 0 pmax ...: pmax + (pmax - mid) / 2 and -mid * wL / 64
            "bdpcm": lambda k, n, l: pmax if k % 2 else 0,
            "mip_a": lambda k, n, l: mid if k <= 0 else (pmax if k <= n // 2 else 0) ^ (pmax if l else 0),   # above: pmax then 0; left: 0 then pmax
            "mip_b": lambda k, n, l: mid if k <= 0 else (0 if k <= n // 2 else pmax) ^ (pmax if l else 0),
            "flat": lambda k, n, l: v, "pad": lambda k, n, l: v}[kind]


def _intra_paint(plane, x, y, w, h, gap, pattern):
    """Writes a block's reference footprint: `gap` identical rows above (corner, then 2w samples) and `gap` identical columns to the left (corner,
    then 2h samples); the MRL corner samples continue the pattern at k < 0."""
    top = np.array([pattern(k, w, 0) for k in range(1 - gap, 2 * w + 1)], np.int16)
    left = np.array([pattern(k, h, 1) for k in range(1 - gap, 2 * h + 1)], np.int16)
    x0, y0 = max(0, x - gap), max(0, y - gap)                      # at the picture's edges only the part inside the picture
    for d in range(gap):
        if y - 1 - d >= 0: row = plane[y - 1 - d, x0:x + 2 * w]; row[:] = top[x0 - x + gap:][:len(row)]
        if x - 1 - d >= 0: col = plane[y0:y + 2 * h, x - 1 - d]; col[:] = left[y0 - y + gap:][:len(col)]
    plane[y0:y, x0:x] = pattern(0, 0, 0)


def _intra_targets_blocks(C, chroma):
    """(comp, w, h, mode, mrl, mip, nb, pattern, v, where) of a targets case with luma CTU size C: cubic modes with MRL 0 / 1 / 2 on every luma shape
    (MRL never on a block as high as the CTU: it could only sit on the CTU's first row), modes 18 / 50 on every shape (PDPC), every MIP mode of every
    shape, transposed and not, BDPCM H / V up to 32x32; per shape a block without neighbours and blocks padded from one unit at 0 and at pmax, and
    one more at the picture's top edge (no neighbour, or the unit left) and one at its left edge (no neighbour, or the unit above), alternating by shape."""
    A = abi
    out = []
    shapes = [(k, 0, w, h) for k, (w, h) in enumerate(INTRA_LUMA_SHAPES) if w <= C and h <= C]
    if chroma: shapes += [(k, c, w, h) for c in (1, 2) for k, (w, h) in enumerate(INTRA_CHROMA_SHAPES) if w <= C // 2 and h <= C // 2]
    for (k, c, w, h) in shapes:                                      # Cr repeats the blocks of Cb: it takes their positions, in its own plane
        if c == 0:
            for mrl in (0, 1, 2):
                if mrl and h == C: continue
                out += [(c, w, h, m, mrl, 0, "full", "cubic", 0, "inner" if mrl else "any") for m in intra_cubic_modes(w, h, mrl)]
            out += [(c, w, h, A.INTRA_MIP, 0, m | (tr << 7), "full", p, 0, "any") for m in range(intra_mip_modes(w, h)) for tr in (0, 1) for p in ("mip_a", "mip_b")]
            if w <= 32 and h <= 32: out += [(c, w, h, m, 0, 0, "full", "bdpcm", 0, "any") for m in (A.INTRA_BDPCM_HOR, A.INTRA_BDPCM_VER)]
        out += [(c, w, h, m, 0, 0, "full", "pdpc", 0, "any") for m in (18, 50)]
        out += [(c, w, h, (1, 66, 2)[k % 3], 0, 0, "none", None, 0, "any"),
                (c, w, h, 50, 0, 0, "one_above", "pad", "0", "any"), (c, w, h, 18, 0, 0, "one_left", "pad", "max", "any"),
                (c, w, h, 1, 0, 0, "one_above", "pad", "max", "any"), (c, w, h, 0, 0, 0, "one_left", "pad", "0", "any")]
        out += [(c, w, h, 0, 0, 0, "none", None, 0, "top_edge") if k & 1 else (c, w, h, 66, 0, 0, "one_left", "pad", "max", "top_edge"),
                (c, w, h, 1, 0, 0, "none", None, 0, "left_edge") if k & 1 else (c, w, h, 2, 0, 0, "one_above", "pad", "0", "left_edge")]
    return out


def _intra_flat_blocks(C, chroma):
    """(comp, w, h, mode, mrl, mip, nb, pattern, v, where) of a flat case: every shape with planar, DC, every angular mode, MRL 1 and 2 with every
    third angular mode (luma), BDPCM H / V (luma up to 32x32); v and the neighbourhood (full, above-right cut, below-left cut) rotate over the blocks."""
    A = abi
    out = []
    shapes = [(0, w, h) for (w, h) in INTRA_LUMA_SHAPES if w <= C and h <= C]
    if chroma: shapes += [(c, w, h) for c in (1, 2) for (w, h) in INTRA_CHROMA_SHAPES if w <= C // 2 and h <= C // 2]
    for (c, w, h) in shapes:
        ms = [(m, 0) for m in range(67)]
        if c == 0: ms += [(m, mrl) for mrl in (1, 2) for m in range(1 + mrl, 67, 3) if h < C] + ([(A.INTRA_BDPCM_HOR, 0), (A.INTRA_BDPCM_VER, 0)] if w <= 32 and h <= 32 else [])
        for i, (m, mrl) in enumerate(ms):
            out.append((c, w, h, m, mrl, 0, ("full", "cut_above", "cut_left")[i % 3], "flat", ("0", "1", "mid", "max-1", "max")[(i + w + h) % 5], "inner" if mrl else "any"))
    return out


def _intra_value(v, bd):
    pmax = (1 << bd) - 1
    return {"0": 0, "1": 1, "mid": 1 << (bd - 1), "max-1": pmax - 1, "max": pmax}[v] if isinstance(v, str) else v


def _intra_record(c, x, y, w, h, mode, mrl, mip, nb):
    A = abi
    unit = 2 if c else 4
    r = np.zeros((), A.INTRA_TU_DTYPE)
    r["x"], r["y"], r["log2w"], r["log2h"], r["comp"], r["mode"], r["multiRefIdx"], r["mip"] = x, y, int(np.log2(w)), int(np.log2(h)), c, mode, mrl, mip
    na, nl = {"full": (2 * w // unit, 2 * h // unit), "cut_above": (w // unit, 2 * h // unit), "cut_left": (2 * w // unit, h // unit),
              "none": (0, 0), "one_above": (1, 0), "one_left": (0, 1)}[nb]
    fl = A.INTRA_ADD_RESI | (A.INTRA_AVAIL_TL if nb == "full" else 0)
    if c == 0 and mode <= 66 and intra_filter_ref(w, h, mode, mrl, 0): fl |= A.INTRA_FILTER_REF
    r["flags"], r["numAbove"], r["numLeft"] = fl, na, nl
    return r


def _intra_chained(ctu, bd):
    """Consumers at CTU (k + 1, 1), k = 0..n - 1, each 16x16 unless noted, each after the producer that writes one of its far reference units, every
    producer a 4x4 (8x4) DC block whose own references are flat at 0 or pmax (its below-left unit is not available): mode 34 at the CTU's top-left corner, its corner in the CTU above-left;
    mode 66 at the top of the CTU, its last above-right unit in the CTU above; mode 66 at the CTU's top right, its last above-right unit in the CTU
    above-right; mode 2 at the CTU's left edge, its last below-left unit in the CTU to the left; an 8x8 mode 45 block with MRL 2 inside the CTU, its
    three reference rows written by an 8x4 producer of the same CTU.  Tags: (role, what, k)."""
    A = abi
    n_ctu = 4
    W, H = (n_ctu + 2) * ctu, 3 * ctu
    recs, tags = [], []
    paints = []                                                   # (x, y, w, h, value) of each producer's reference footprint
    for k in range(n_ctu):
        X, Y = (k + 1) * ctu, ctu
        v = (k & 1) * ((1 << bd) - 1)
        cons = [(X, Y, 16, 16, 34, 0, "corner"), (X + 24, Y, 16, 16, 66, 0, "above"), (X + ctu - 16, Y, 16, 16, 66, 0, "above_right"),
                (X, Y + 16, 16, 16, 2, 0, "below_left"), (X + 48, Y + 24, 8, 8, 45, 2, "mrl2")]      # in decoding order: no block reads a later one
        prods = {"above_right": [(X + ctu + 12, Y - 4, 4, 4)], "below_left": [(X - 4, Y + 44, 4, 4)], "corner": [(X - 4, Y - 4, 4, 4)],
                 "above": [(X + 52, Y - 4, 4, 4)], "mrl2": [(X + 48, Y + 20, 8, 4)]}
        for (x, y, w, h, mode, mrl, what) in cons:
            for (px, py, pw, ph) in prods[what]:
                pv = ((1 << bd) - 1) - v if what in ("corner", "mrl2") else v
                r = _intra_record(0, px, py, pw, ph, 1, 0, 0, "cut_left")     # its below-left is a later block: not available
                recs.append(r); tags.append(("producer", what, k)); paints.append((px, py, pw, ph, pv))
            recs.append(_intra_record(0, x, y, w, h, mode, mrl, 0, "full")); tags.append(("consumer", what, k))
    recs = np.array(recs, A.INTRA_TU_DTYPE)
    key = (recs["y"].astype(int) // ctu) * (W // ctu) + recs["x"].astype(int) // ctu
    order = np.argsort(key, kind="stable")
    return W, H, recs[order], [tags[i] for i in order], paints


_intra_sweep_cache = {}


def intra_designed_sweep(name):
    """One case of the designed regular intra sweep (INTRA_SWEEP_CASES) as a dict: geometry (g, W, H, bd, ctu), noise planes with the designed
    references written in (planes; Cb / Cr None in 4:0:0), the residual planes (resi), the records in CTU order (recs) and per record what it was built
    for (tags: (pattern, value, neighbourhood, where), or the chained role); flat: the value every predicted sample of a record must hold (-1: none)."""
    if name in _intra_sweep_cache: return _intra_sweep_cache[name]
    kind, ctu, bd, pad, chroma = INTRA_SWEEP_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    pmax = (1 << bd) - 1
    if kind == "chained":
        W, H, recs, tags, paints = _intra_chained(ctu, bd)
        planes = noise_planes(rng, W, H, bd)
        for (x, y, w, h, v) in paints: _intra_paint(planes[0], x, y, w, h, 4, _intra_pattern("flat", bd, v))
        flat = np.full(len(recs), -1)
    else:
        blocks = _intra_targets_blocks(ctu, chroma) if kind == "targets" else _intra_flat_blocks(ctu, chroma)
        ctus_w = max(8, 2048 // ctu)
        luma = [i for i, b in enumerate(blocks) if b[0] == 0]
        cb = [i for i, b in enumerate(blocks) if b[0] == 1]
        cr = [i for i, b in enumerate(blocks) if b[0] == 2]
        pos = {}
        for i, p in zip(luma, _cclm_pack([(blocks[i][1], blocks[i][2], blocks[i][9]) for i in luma], ctu, ctus_w, gap=4)): pos[i] = p
        for i, p in zip(cb, _cclm_pack([(blocks[i][1], blocks[i][2], blocks[i][9]) for i in cb], ctu // 2, ctus_w, gap=2)): pos[i] = p
        for i, j in zip(cr, cb): pos[i] = pos[j]                  # Cr blocks sit where the Cb blocks of the same list position sit, in their own plane
        assert all(blocks[i][1:3] == blocks[j][1:3] for i, j in zip(cr, cb))
        W = ctus_w * ctu
        H = ((max((y + 2 * blocks[i][2]) << (blocks[i][0] > 0) for i, (x, y) in pos.items()) + ctu - 1) // ctu + 1) * ctu
        strides = (W + pad, W // 2 + pad, W // 2 + pad) if pad else None
        planes = noise_planes(rng, W, H, bd, chroma=chroma, strides=strides)
        per = []
        for i, b in enumerate(blocks):
            c, w, h, mode, mrl, mip, nb, pattern, v, where = b
            x, y = pos[i]
            if pattern: _intra_paint(planes[c], x, y, w, h, 2 if c else 4, _intra_pattern(pattern, bd, _intra_value(v, bd)))
            per.append((_intra_record(c, x, y, w, h, mode, mrl, mip, nb), (pattern, v, nb, where), _intra_value(v, bd) if pattern == "flat" else -1))
        key = [((int(r["y"]) << (r["comp"] > 0)) // ctu) * (W // ctu) + ((int(r["x"]) << (r["comp"] > 0)) // ctu) for r, _, _ in per]
        order = np.argsort(key, kind="stable")
        recs = np.array([per[i][0] for i in order], abi.INTRA_TU_DTYPE)
        tags = [per[i][1] for i in order]
        flat = np.array([per[i][2] for i in order])
    g = abi.make_geom(W, H, bd, chroma_format=1 if chroma else 0, ctu=ctu, strides=tuple(p.shape[1] for p in planes) if chroma else (planes[0].shape[1], 0, 0))
    lim = (3 * pmax) // 4 if kind != "flat" else 64
    resi = [rng.integers(-lim, lim + 1, size=p.shape).astype(np.int16) for p in planes]
    if not chroma: planes, resi = planes + [None, None], resi + [None, None]
    case = dict(name=name, g=g, W=W, H=H, bd=bd, ctu=ctu, planes=planes, resi=resi, recs=recs, tags=tags, flat=flat)
    _intra_sweep_cache[name] = case
    return case


# ---------------------------------------------------------------------------------------------------------------- designed K2 sweep
# A fixed list of named K2 cases (tests/test_k2_*.py): every PU shape under every tool it allows, every 1/16 luma phase pair in each tile list, tiles whose
# reference windows sit on the interior / boundary thresholds of k2_inter.cu, MVs at the clipMv bounds and at +-2^17, and reference content built so that
# DMVR's search provably ends where the case says.  Nothing is drawn at random except the noise of the reference pictures, from a seed fixed per case.
MC_SIZES = (4, 8, 16, 32, 64, 128)
MC_AFFINE_TOOLS = tuple(f"aff{n}_{d}{p}" for n in (4, 6) for d in ("uni", "bi") for p in ("", "_prof"))
MC_TOOLS = ("uni0", "uni1", "bi", "bcw-2", "bcw3", "bcw5", "bcw10", "bdof", "dmvr", "dmvr_bdof", "althpel") + MC_AFFINE_TOOLS + ("geo",)
MC_WP_TOOLS = ("wp_uni0", "wp_uni1", "wp_bi", "wp_aff4_uni", "wp_aff6_bi_prof")
MC_LISTS = [(m, k) for m in range(4) for k in range(4) if m < 2 or k >= 2]       # the 12 translational (mode, size class) lists; 16 = affine


def mc_tool_legal(tool, w, h):
    """The shapes VVC allows a tool at (bucket.cu pu_head and InterPrediction.cpp:1372-1420): no bi-prediction for 4x4, 4x8 and 8x4; BCW from 256
    samples; BDOF / DMVR from 8x8 and 128 samples; affine from 8x8; GEO 8..64 per side with an aspect ratio of at most 4.  A CU 128 samples wide or
    high is at least 64 samples in the other direction (the 64x64 pipeline units forbid splitting a 128x64 CU further across its long side)."""
    if max(w, h) == 128 and min(w, h) < 64: return False
    big = w >= 8 and h >= 8 and w * h >= 128
    t = tool[3:] if tool.startswith("wp_") else tool
    if t in ("uni0", "uni1", "althpel"): return True
    if t == "bi": return w + h > 12
    if t.startswith("bcw"): return w * h >= 256
    if t in ("bdof", "dmvr", "dmvr_bdof"): return big
    if t.startswith("aff"): return w >= 8 and h >= 8
    if t == "geo": return 8 <= w <= 64 and 8 <= h <= 64 and w < 8 * h and h < 8 * w
    raise ValueError(tool)


def mc_list_of(pu, tx, ty):
    """bucket.cu mc_list_of: the list of luma tile (tx, ty) of a PU, mode * 4 + size class (32 / 64 / 128 / 256 samples), 16 = affine."""
    f, w, h = int(pu["flags"]), int(pu["w"]), int(pu["h"])
    if f & PU_AFFINE: return 16
    bi = pu["refSlot"][0] >= 0 and pu["refSlot"][1] >= 0
    mode = 1 if f & PU_GEO else 3 if f & PU_DMVR else 2 if bi and f & PU_BDOF else 1 if bi else 0
    n = min(16, w - 16 * tx) * min(16, h - 16 * ty)
    return mode * 4 + (0 if n <= 32 else 1 if n <= 64 else 2 if n <= 128 else 3)


def mc_tiles(pus):
    """Every luma tile of a PU list: (PU index, tx, ty, list)."""
    return [(i, tx, ty, mc_list_of(p, tx, ty)) for i, p in enumerate(pus) for ty in range((int(p["h"]) + 15) // 16) for tx in range((int(p["w"]) + 15) // 16)]


def mc_affine_over(pu, l):
    """k2_inter.cu spread_over_limit / aff_model for list l of an affine PU (InterPrediction.cpp:1001-1030): the sub-block MVs collapse to the
    centre MV and PROF is off when the spread of the 4x4 sub-block footprint is over the memory-bandwidth limit."""
    l2w, l2h = int(pu["w"]).bit_length() - 1, int(pu["h"]).bit_length() - 1
    LT, RT, LB = [int(v) for v in pu["mv"][l]], [int(v) for v in pu["cpmv"][l][0]], [int(v) for v in pu["cpmv"][l][1]]
    a, b = (RT[0] - LT[0]) << (7 - l2w), (RT[1] - LT[1]) << (7 - l2w)
    if pu["flags"] & PU_AFFINE6: c, d = (LB[0] - LT[0]) << (7 - l2h), (LB[1] - LT[1]) << (7 - l2h)
    else: c, d = -b, a
    s4, ft = 4 << 11, 6
    if pu["interDir"] == 3:
        xs, ys = (0, 4 * a + s4, 4 * c, 4 * a + 4 * c + s4), (0, 4 * b, 4 * d + s4, 4 * b + 4 * d + s4)
        return (((max(xs) - min(xs)) >> 11) + ft + 3) * (((max(ys) - min(ys)) >> 11) + ft + 3) > (ft + 9) * (ft + 9)
    rw, rh = ((max(0, 4 * a + s4) - min(0, 4 * a + s4)) >> 11) + ft + 3, ((max(0, 4 * b) - min(0, 4 * b)) >> 11) + ft + 3
    if rw * rh > (ft + 9) * (ft + 5): return True
    rw, rh = ((max(0, 4 * c) - min(0, 4 * c)) >> 11) + ft + 3, ((max(0, 4 * d + s4) - min(0, 4 * d + s4)) >> 11) + ft + 3
    return rw * rh > (ft + 5) * (ft + 9)


def _mc_pu(x, y, w, h, slots, mv0=(0, 0), mv1=(0, 0), flags=0, bcw=4, cpmv=None):
    r = np.zeros((), PU_DTYPE)
    r["x"], r["y"], r["w"], r["h"], r["flags"], r["bcwW1"] = x, y, w, h, flags, bcw
    r["refSlot"] = slots
    r["interDir"] = 3 if slots[0] >= 0 and slots[1] >= 0 else 1 if slots[0] >= 0 else 2
    r["mv"] = (mv0, mv1)
    if cpmv is not None: r["cpmv"] = cpmv
    return r


def _mc_mv(k, salt=0):
    """MV number k of a cycle: phase pair (k * 7 + salt) mod 256 of the 16 x 16 luma phases, and with it both values of the extra chroma phase bit
    (so every 1/32 chroma phase), integer part -4..4 / -3..3 samples."""
    i = (k * 7 + salt) % 256
    fx, fy = i % 16, i // 16
    ax, ay = (k * 5 + salt) % 9 - 4, (k * 3 + salt) % 7 - 3
    return (ax * 32 + ((i >> 4) & 1) * 16 + fx, ay * 32 + (i & 1) * 16 + fy)


def _mc_tool_pu(tool, x, y, w, h, k):
    """The PU of `tool` at (x, y, w, h), k-th of its kind (k cycles the phases, the reference slots and the affine / GEO parameters)."""
    mv0, mv1 = _mc_mv(k), _mc_mv(k, 101)
    p = k & 1
    t = tool[3:] if tool.startswith("wp_") else tool
    if t == "uni0": return _mc_pu(x, y, w, h, (p, -1), mv0)
    if t == "uni1": return _mc_pu(x, y, w, h, (-1, 2 + p), mv0, mv1)
    if t in ("bi", "bi_small"): return _mc_pu(x, y, w, h, (p, 2 + ((k >> 1) & 1)), mv0, mv1)
    if t.startswith("bcw"): return _mc_pu(x, y, w, h, (p, 2 + ((k >> 1) & 1)), mv0, mv1, bcw=int(t[3:]))
    if t == "bdof": return _mc_pu(x, y, w, h, (p, 2 + p), mv0, mv1, PU_BDOF)
    if t in ("dmvr", "dmvr_bdof"): return _mc_pu(x, y, w, h, (p, 2 + p), mv0, mv1, PU_DMVR | (PU_BDOF if t == "dmvr_bdof" else 0))
    if t == "althpel":                                          # AMVR half-pel: MVs in half samples, the 6-tap half-sample filter; chroma 0, 8, 16, 24 / 32
        a0, a1 = (8 * ((k % 4) - 2), 8 * ((k // 4) % 4 - 2)), (8 * ((k * 3) % 8 - 4), 8 * ((k * 5 + 1) % 8 - 3))
        return _mc_pu(x, y, w, h, (p, 2 + p) if w + h > 12 else (p, -1), a0, a1, PU_ALTHPEL)
    if t.startswith("aff"):
        six, bi, prof = t.startswith("aff6"), "_bi" in t, t.endswith("_prof")
        d = [(((k * 13 + 7 * l) % 49) - 24, ((k * 29 + 3 * l) % 49) - 24) for l in range(4)]
        cp = [[(mv0[0] + d[0][0], mv0[1] + d[0][1]), (mv0[0] + d[1][0], mv0[1] + d[1][1])], [(mv1[0] + d[2][0], mv1[1] + d[2][1]), (mv1[0] + d[3][0], mv1[1] + d[3][1])]]
        fl = PU_AFFINE | (PU_AFFINE6 if six else 0) | (PU_PROF0 | PU_PROF1 if prof else 0)
        return _mc_pu(x, y, w, h, (p, 2 + p) if bi else ((p, -1) if k & 2 else (-1, 2 + p)), mv0, mv1, fl, cpmv=cp)
    if t == "geo": return _mc_pu(x, y, w, h, (k % 4, (k * 3 + 1) % 4), mv0, mv1, PU_GEO, bcw=k % 64)
    raise ValueError(tool)


def _mc_pack(sizes, W, gap=0, margin=0):
    """Shelf packing of (w, h) rectangles (powers of two) into a picture W wide, tallest first.  Every block starts at a multiple of its own size, so no
    block crosses a CTU boundary (a CU never does; the reference keeps motion per CTU).  Returns (positions, height used)."""
    order = sorted(range(len(sizes)), key=lambda i: (-sizes[i][1], -sizes[i][0], i))
    up = lambda v, a: (v + a - 1) // a * a
    pos = [None] * len(sizes); x = margin; y = margin; rowh = 0
    for i in order:
        w, h = sizes[i]
        if up(x, w) + w > W - margin or rowh == 0:
            y = up(y + rowh + (gap if rowh else 0), h); x = margin; rowh = h
        x = up(x, w)
        pos[i] = (x, y); x += w + gap
    return pos, y + rowh + margin


def _mc_finish(pus):
    """dmvrOff of the DMVR PUs (one entry per 16x16 sub-block), the list as an array, the number of entries."""
    pus = np.array(pus, PU_DTYPE)
    off = 0
    for p in pus:
        if p["flags"] & PU_DMVR:
            p["dmvrOff"] = off; off += max(1, int(p["w"]) >> 4) * max(1, int(p["h"]) >> 4)
    return pus, off


def mc_shape_tool_specs(tools=MC_TOOLS, bd=10):
    """(tool, w, h) of every legal shape x tool pair (DMVR only up to 10 bit); GEO: the 64 split directions spread over its 14 shapes; plus the bi-predicted
    4x8 / 8x4 blocks ('bi_small'): the standard never codes them, but the PU list accepts them and they are what fills the 32-sample bi list."""
    out = []
    for t in tools:
        if t.endswith("geo"): continue
        if bd > 10 and "dmvr" in t: continue
        out += [(t, w, h) for h in MC_SIZES for w in MC_SIZES if mc_tool_legal(t, w, h)]
    if "geo" in tools:
        shapes = [(w, h) for h in MC_SIZES for w in MC_SIZES if mc_tool_legal("geo", w, h)]
        out += [("geo", *shapes[d % len(shapes)]) for d in range(64)]
        out += [("bi_small", 8, 4), ("bi_small", 4, 8)]
    return out


def _mc_shapes_case(W, specs, gap=0, ctu=128):
    """The PUs of (tool, w, h) specs no larger than the CTU, packed into a picture W wide, the k-th of each tool with the k-th MV of its cycle."""
    specs = [s for s in specs if max(s[1], s[2]) <= ctu]
    pos, used = _mc_pack([(w, h) for _, w, h in specs], W, gap=gap)
    count, pus, tags = {}, [], []
    for (t, w, h), (x, y) in zip(specs, pos):
        k = count.get(t, 0); count[t] = k + 1
        pus.append(_mc_tool_pu(t, x, y, w, h, k)); tags.append(t)
    return pus, tags, used


def _mc_phase_case(W):
    """256 single-tile PUs per translational list, one per luma phase pair of list 0 (list 1 cycles independently), + AltHpel PUs of every class."""
    shape = {0: (8, 4), 1: (8, 8), 2: (16, 8), 3: (16, 16)}
    tool = {0: "uni0", 1: "bi", 2: "bdof", 3: "dmvr"}
    specs = []
    for (m, c) in MC_LISTS:
        t = "bi_small" if (m, c) == (1, 0) else tool[m]
        specs += [(t, *shape[c], (m, c), k) for k in range(256)]
    specs += [("althpel", *shape[c], None, k) for c in range(4) for k in range(16)]
    pos, used = _mc_pack([(w, h) for _, w, h, _, _ in specs], W)
    pus, tags = [], []
    for (t, w, h, lst, k), (x, y) in zip(specs, pos):
        pu = _mc_tool_pu(t, x, y, w, h, k)
        if lst is not None:                                    # phase pair k exactly (the integer part still cycles)
            mv = _mc_mv(k); fx, fy = k % 16, k // 16
            pu["mv"][0] = ((mv[0] & ~15) | fx, (mv[1] & ~15) | fy)
        pus.append(pu); tags.append(t)
    return pus, tags, used


# ---- windows of a tile (k2_inter.cu): the integer reference position of its first sample, and the interior tests
def mc_tile_windows(pu, l, tx=0, ty=0):
    """Integer reference positions of tile (tx, ty) of a PU for list l before any clipping: luma (ox, oy), chroma (ocx, ocy) as the uni / bi / BDOF tiles
    compute them (mc_tile, motion per list), and the DMVR search origins (ix, iy), (icx, icy) (dmvr_search)."""
    bx, by = int(pu["x"]) + 16 * tx, int(pu["y"]) + 16 * ty
    mx, my = int(pu["mv"][l][0]), int(pu["mv"][l][1])
    return dict(luma=(bx + (mx >> 4), by + (my >> 4)), chroma=((bx >> 1) + (mx >> 5), (by >> 1) + (my >> 5)),
                dmvr=(bx + (mx >> 4), by + (my >> 4)), dmvr_chroma=((bx >> 1) + (mx >> 5), (by >> 1) + (my >> 5)))


def mc_window_margins(kind, W, H, tw, th):
    """For a window kind, (first interior x, last interior x, first interior y, last interior y) of its origin: the stage A predicates of k2_inter.cu
    mc_tile (luma / chroma footprints of the 8- / 4-tap filters) and the search-window predicates of dmvr_search."""
    cw, ch, CW, CH = tw >> 1, th >> 1, W >> 1, H >> 1
    if kind == "luma": return 4, W - tw - 5, 3, H - th - 4
    if kind == "chroma": return 2, CW - cw - 3, 1, CH - ch - 2
    if kind == "dmvr": return 6, W - tw - 9, 6, H - th - 9
    if kind == "dmvr_chroma": return 4, CW - cw - 6, 3, CH - ch - 5
    raise ValueError(kind)


def _mc_edge_specs(chroma, bd):
    """Single-tile PUs of one shape per translational list x window kind x edge x offset (-1, 0, +1 around the first interior position)."""
    shape = {(0, 0): (8, 4), (0, 1): (8, 8), (0, 2): (16, 8), (0, 3): (16, 16), (1, 0): (4, 8), (1, 1): (8, 8), (1, 2): (8, 16), (1, 3): (16, 16),
             (2, 2): (16, 8), (2, 3): (16, 16), (3, 2): (8, 16), (3, 3): (16, 16)}
    tool = {0: "uni0", 1: "bi", 2: "bdof", 3: "dmvr_bdof"}
    out = []
    for (m, c) in MC_LISTS:
        if m == 3 and bd > 10: continue
        kinds = ("dmvr",) + (("dmvr_chroma",) if chroma else ()) if m == 3 else ("luma",) + (("chroma",) if chroma else ())
        for kind in kinds:
            for edge in "lrtb":
                for off in (-1, 0, 1):
                    out.append(("bi_small" if (m, c) == (1, 0) else tool[m], *shape[(m, c)], kind, edge, off))
    return out


def _mc_edges_case(W, H, ctu, chroma, bd):
    """Threshold tiles (see _mc_edge_specs), PUs with MVs at the clipMv bounds of this CTU size and one sample past them, and MVs near +-2^17.  The
    affine ones among the latter have sub-block MVs past the +-2^17 storage clamp.  The DMVR ones do not make the refinement cross that clamp
    (the clamp of the refined MV in k2_inter.cu dmvr_search): both search windows lie wholly outside the picture, where every sample replicates the
    border, so the search ends at the centre with a zero delta.  No picture narrower than 2^13 samples can do otherwise, and clipMv follows the clamp in any case."""
    specs = _mc_edge_specs(chroma, bd)
    tools = ("uni0", "bi", "aff4_uni_prof") + (("dmvr_bdof",) if bd <= 10 else ())
    bounds = ("xlo", "xlo-1", "xhi", "xhi+1", "ylo", "ylo-1", "yhi", "yhi+1")
    clip = [(tools[(i + j) % len(tools)], s, s, b) for i, b in enumerate(bounds) for j, s in enumerate((32, 64, 128) if i % 2 == 0 else (32, 64)) if s <= ctu]
    far = [(t, 16, 16, s) for t in ("uni0", "bi", "aff4_bi", "aff6_uni_prof") + (("dmvr", "dmvr_bdof") if bd <= 10 else ()) for s in (1, -1)]
    sizes = [(w, h) for _, w, h, *_ in specs] + [(w, h) for _, w, h, _ in clip] + [(w, h) for _, w, h, _ in far]
    pos, used = _mc_pack(sizes, W)
    assert used <= H, (used, H)
    pus, tags, marks = [], [], []
    for k, ((t, w, h, kind, edge, off), (x, y)) in enumerate(zip(specs, pos)):
        pu = _mc_tool_pu(t, x, y, w, h, k)
        bi = pu["refSlot"][0] >= 0 and pu["refSlot"][1] >= 0
        l = (k & 1) if bi else 0                               # the list that sits on the threshold; the other one looks at the centre
        x0, x1, y0, y1 = mc_window_margins(kind, W, H, w, h)
        sh = 5 if kind in ("chroma", "dmvr_chroma") else 4
        bx, by = (x >> 1, y >> 1) if sh == 5 else (x, y)
        tx_, ty_ = (x0 + x1) // 2, (y0 + y1) // 2
        if edge == "l": tx_ = x0 + off
        if edge == "r": tx_ = x1 + off
        if edge == "t": ty_ = y0 + off
        if edge == "b": ty_ = y1 + off
        f = int(pu["mv"][l][0]) & ((1 << sh) - 1), int(pu["mv"][l][1]) & ((1 << sh) - 1)
        pu["mv"][l] = (((tx_ - bx) << sh) + f[0], ((ty_ - by) << sh) + f[1])
        if bi:
            o = 1 - l; cx, cy = W // 2 - w // 2, H // 2 - h // 2
            pu["mv"][o] = (((cx - x) << 4) + (int(pu["mv"][o][0]) & 15), ((cy - y) << 4) + (int(pu["mv"][o][1]) & 15))
        pus.append(pu); tags.append(t); marks.append((len(pus) - 1, kind, edge, off, l))
    n0 = len(specs)
    for k, ((t, w, h, b), (x, y)) in enumerate(zip(clip, pos[n0:n0 + len(clip)])):
        pu = _mc_tool_pu(t, x, y, w, h, k)
        lo = lambda p: (-ctu - 8 - p + 1) * 16
        hi = lambda p, S: (S + 8 - p - 1) * 16
        v = {"xlo": lo(x), "xlo-1": lo(x) - 16, "xhi": hi(x, W), "xhi+1": hi(x, W) + 16,
             "ylo": lo(y), "ylo-1": lo(y) - 16, "yhi": hi(y, H), "yhi+1": hi(y, H) + 16}[b] + (k % 5) * 3
        for l in range(2):
            mv = [int(pu["mv"][l][0]), int(pu["mv"][l][1])]
            mv[0 if b[0] == "x" else 1] = v
            if t.startswith("aff"): pu["cpmv"][l] = pu["cpmv"][l] - pu["mv"][l] + mv
            pu["mv"][l] = mv
        pus.append(pu); tags.append(t); marks.append((len(pus) - 1, "clip", b, 0, 0))
    n1 = n0 + len(clip)
    for k, ((t, w, h, s), (x, y)) in enumerate(zip(far, pos[n1:])):
        pu = _mc_tool_pu(t, x, y, w, h, k)
        m = (1 << 17) - 1
        mv0, mv1 = (s * m - s * 9, -s * m + s * 12), (-s * m + s * 7, s * m - s * 20)
        if t.startswith("aff"): pu["cpmv"] = [[(mv0[0] + 400 * s, mv0[1]), (mv0[0], mv0[1] + 300 * s)], [(mv1[0] - 400 * s, mv1[1] + 200), (mv1[0], mv1[1] - 300 * s)]]
        pu["mv"] = (mv0, mv1)
        pus.append(pu); tags.append(t); marks.append((len(pus) - 1, "far", "+" if s > 0 else "-", 0, 0))
    return pus, tags, marks


def _mc_affine_case(W, ctu):
    """Affine PUs with CPMV spreads one step under and one step over the bandwidth limit (4- / 6-parameter, uni / bi, PROF on), equal CPMVs (PROF off
    whatever the flag says), in every affine size class."""
    specs = []
    for (w, h) in ((8, 8), (16, 16), (32, 16), (16, 64), (64, 64), (128, 64)):
        for six in (0, 1):
            for bi in (0, 1):
                for side in ("under", "over", "equal"):
                    if max(w, h) <= ctu: specs.append((w, h, six, bi, side, (len(specs) // 3) & 1))
    pos, used = _mc_pack([(w, h) for w, h, *_ in specs], W)
    pus, tags = [], []
    for k, ((w, h, six, bi, side, dirn), (x, y)) in enumerate(zip(specs, pos)):
        t = f"aff{6 if six else 4}_{'bi' if bi else 'uni'}_prof"
        pu = _mc_tool_pu(t, x, y, w, h, k)
        for l in range(2):
            base = np.array(pu["mv"][l], np.int64)
            if side == "equal":
                pu["cpmv"][l] = (base, base); continue
            step = 0
            def with_step(s):
                q = pu.copy()
                d = (s, 0) if dirn == 0 else (0, s)
                q["cpmv"][l] = (base + d, base + ((0, s) if six and dirn == 0 else (s, 0) if six else (0, 0)))
                return q
            while not mc_affine_over(with_step(step + 1), l) and step < 4000: step += 1
            pu["cpmv"][l] = with_step(step + (1 if side == "over" else 0))["cpmv"][l]
        pus.append(pu); tags.append(t)
    return pus, tags, used


def _mc_dmvr_target_case(W):
    """DMVR PUs whose mirrored search provably ends on a chosen one of the 25 integer positions: slots 2 / 3 are copies of slots 0 / 1 (slot 3 shifted by
    (3, -2) samples), so that list 1's MV is list 0's + 2 * target - shift and the SAD is zero exactly there.  Centre targets stand for the early exit."""
    shapes = [(16, 16), (8, 16), (16, 8), (32, 16), (16, 32), (64, 64)]
    specs = [(d, shapes[(d + j) % len(shapes)], j) for d in range(25) for j in range(3)] + [(d, (128, 128), 0) for d in (3, 21)]
    pos, used = _mc_pack([s for _, s, _ in specs], W, gap=4, margin=32)
    pus, tags, targets = [], [], []
    for k, ((d, (w, h), j), (x, y)) in enumerate(zip(specs, pos)):
        u, v = d % 5 - 2, d // 5 - 2
        p = k & 1
        s = (0, 0) if p == 0 else (3, -2)
        mv0 = _mc_mv(k); mv0 = ((mv0[0] & 15) + 16 * ((k % 5) - 2), (mv0[1] & 15) + 16 * ((k % 3) - 1))
        mv1 = (mv0[0] + 16 * (2 * u - s[0]), mv0[1] + 16 * (2 * v - s[1]))
        pus.append(_mc_pu(x, y, w, h, (p, 2 + p), mv0, mv1, PU_DMVR | (PU_BDOF if j != 1 else 0))); tags.append("dmvr_target")
        targets.append((len(pus) - 1, u, v))
    return pus, tags, targets, used


# designed DMVR cost surfaces (content along x or y only, integer MVs): name -> (pattern, expected delta); see _mc_paint
MC_DMVR_SURFACES = {
    "tie_minus8_x": (-8, 0), "tie_plus8_x": (8, 0), "tie_minus8_y": (0, -8), "tie_plus8_y": (0, 8),     # a neighbour's SAD equals the scaled centre cost
    "den0_x": (0, 0), "den0_y": (0, 0),                                                                  # both neighbours equal it: the surface is flat
    "den0_x_bio_off": (0, 0),                                                                            # the same with minCost in [tw*th, 2*tw*th): BDOF off
    "den0_x_ramp_y_bio_off": (0, 5),       # + a vertical ramp of 3 per row in both lists: the y surface is no longer flat, and BDOF would change samples
    "flat_exit": (0, 0),                                                                                 # identical flat windows: SAD 0, the early exit
}


def _mc_paint(kind, A, B, x0, y0, w, h):
    """Paints the windows of a PU at (x0, y0) in slot planes A (list 0) and B (list 1), 8 samples beyond the block on every side.
    tie_*: A is a ramp of slope 7, B = A -+ 8, so that the SAD of shift u is N |14u +- 8|: u = -+1 costs 6N = the centre's 8N scaled by 3/4, and the strict
    raster-order search keeps the centre, with an equal neighbour.  den0_*: A has period 4 (0 0 K K), B = A shifted by 2 plus c = 3K/4: odd shifts cost
    c N = 3/4 of the centre's K N, even ones K N."""
    ys, xs = np.mgrid[y0 - 8:y0 + h + 8, x0 - 8:x0 + w + 8]
    axis = xs - (x0 - 8) if kind.endswith("_x") or "_x_" in kind else ys - (y0 - 8)
    sl = (slice(y0 - 8, y0 + h + 8), slice(x0 - 8, x0 + w + 8))
    if kind.startswith("tie"):
        a = 16 + 7 * axis
        A[sl] = a; B[sl] = a - 8 if "minus" in kind else a + 8
    elif kind.startswith("den0"):
        K, c = (4, 3) if kind.endswith("bio_off") else (40, 30)
        ramp = 3 * (ys - (y0 - 8)) if "ramp_y" in kind else 0
        A[sl] = 300 + K * ((axis % 4) >= 2) + ramp; B[sl] = 300 + K * (((axis + 2) % 4) >= 2) + c + ramp
    elif kind == "flat_exit":
        A[sl] = 77; B[sl] = 77


def _mc_surface_case(W):
    shapes = [(16, 16), (8, 16), (16, 8), (32, 32), (32, 16)]
    specs = [(kind, s, bdof) for kind in MC_DMVR_SURFACES for s in shapes for bdof in (0, 1)]
    pos, used = _mc_pack([s for _, s, _ in specs], W, gap=24, margin=16)
    pus, tags = [], []
    for (kind, (w, h), bdof), (x, y) in zip(specs, pos):
        pus.append(_mc_pu(x, y, w, h, (0, 2), (0, 0), (0, 0), PU_DMVR | (PU_BDOF if bdof else 0))); tags.append(kind)
    return pus, tags, used


def _mc_refs(name, W, H, bd, chroma, strides, recipe, pus=None, tags=None):
    """The four DPB slots of a case.  recipe: 'noise' (independent noise per slot), 'copies' (slots 2 / 3 = slots 0 / 1, slot 3 rolled by (3, -2)),
    'flat' (one value per slot, slots 0 and 2 equal), 'extreme' (0 / 2^bd-1 checkerboards, stripes and steps), 'surfaces' (painted DMVR cost surfaces)."""
    import zlib
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    pmax = (1 << bd) - 1
    slots = [noise_planes(rng, W, H, bd, chroma=chroma, strides=strides) for _ in range(4)]
    if recipe == "copies":
        slots[2] = [p.copy() for p in slots[0]]
        slots[3] = []
        for c, p in enumerate(slots[1]):
            w = W >> (1 if c else 0); q = p.copy()
            q[:, :w] = np.roll(p[:, :w], (2 >> (1 if c else 0), -3 >> (1 if c else 0)), axis=(0, 1))
            slots[3].append(q)
    elif recipe in ("flat", "surfaces"):
        vals = (bd > 8 and 700 or 180, 300 >> (10 - bd) if bd <= 10 else 1200, bd > 8 and 700 or 180, 5)
        for s in range(4):
            for p in slots[s]: p[...] = vals[s]
    elif recipe == "extreme":
        for s in range(4):
            for c, p in enumerate(slots[s]):
                h, w = p.shape[0], W >> (1 if c else 0)
                yy, xx = np.mgrid[0:h, 0:w]
                pat = [((xx + yy) & 1), ((xx // 3) & 1), ((yy // 2) & 1) ^ ((xx // 5) & 1), (xx >= w // 2 + ((yy * 3) % 7) - 3)][s]
                p[:, :w] = np.where(pat, pmax, 0)
    if recipe == "surfaces":
        for pu, kind in zip(pus, tags):
            _mc_paint(kind, slots[0][0], slots[2][0], int(pu["x"]), int(pu["y"]), int(pu["w"]), int(pu["h"]))
    if not chroma:
        slots = [[s[0], s[0][:1], s[0][:1]] for s in slots]
    return slots


# name -> (W, H, bitDepth, CTU size, 4:2:0?, strides or None, content of the slots, builder)
MC_SWEEP_CASES = {
    "shapes_10bit": (1920, 1080, 10, 128, 1, None, "noise", "shapes"),
    "shapes_8bit_extreme": (1920, 1080, 8, 128, 1, None, "extreme", "shapes"),
    "shapes_12bit_extreme": (1920, 1080, 12, 128, 1, None, "extreme", "shapes"),
    "shapes_10bit_flat": (1920, 1080, 10, 128, 1, None, "flat", "shapes"),
    "shapes_yuv400_10bit": (1920, 1080, 10, 128, 0, None, "noise", "shapes"),
    "phases_10bit": (1920, 400, 10, 128, 1, None, "noise", "phases"),
    "phases_8bit_stride_odd": (1920, 400, 8, 64, 1, (1923, 961, 961), "noise", "phases"),
    "edges_ctu128": (832, 480, 10, 128, 1, None, "noise", "edges"),
    "edges_ctu64_stride_pad": (832, 472, 10, 64, 1, (836, 418, 418), "noise", "edges"),
    "edges_ctu32_stride_odd": (832, 480, 10, 32, 1, (833, 417, 417), "noise", "edges"),
    "edges_ctu32_yuv400_8bit": (832, 456, 8, 32, 0, None, "noise", "edges"),
    "edges_ctu64_12bit_extreme": (832, 472, 12, 64, 1, (840, 420, 420), "extreme", "edges"),
    "affine_limits_10bit": (832, 480, 10, 128, 1, None, "noise", "affine"),
    "affine_limits_12bit_stride_odd": (832, 480, 12, 64, 1, (833, 417, 417), "extreme", "affine"),
    "dmvr_targets_10bit": (1280, 720, 10, 128, 1, None, "copies", "targets"),
    "dmvr_targets_8bit_stride_pad": (1280, 720, 8, 128, 1, (1284, 642, 642), "copies", "targets"),
    "dmvr_surfaces_10bit": (1280, 720, 10, 128, 1, None, "surfaces", "surfaces"),
    "wp_10bit": (1920, 1080, 10, 128, 1, None, "noise", "wp"),
    "wp_12bit_extreme": (1920, 1080, 12, 128, 1, None, "extreme", "wp"),
    "wp_8bit_stride_odd": (1920, 1080, 8, 128, 1, (1921, 961, 961), "noise", "wp"),
}

_mc_sweep_cache = {}


def mc_sweep(name):
    """One case of the designed K2 sweep (MC_SWEEP_CASES) as a dict: geometry (g, W, H, bd, ctu, chroma, strides), the PU list and its number of DMVR
    entries, the DPB slots (refs), the tool / pattern of every PU (tags), explicit weights (wp = (raw, entries)) for the wp cases, threshold marks
    (edges cases: (PU index, window kind, edge, offset, list)) and DMVR targets ((PU index, u, v) for the targets case)."""
    if name in _mc_sweep_cache: return _mc_sweep_cache[name]
    from . import abi as A
    W, H, bd, ctu, chroma, strides, recipe, kind = MC_SWEEP_CASES[name]
    marks, targets, wp = [], [], None
    if kind == "shapes":
        pus, tags, used = _mc_shapes_case(W, mc_shape_tool_specs(bd=bd), ctu=ctu)
    elif kind == "wp":
        pus, tags, used = _mc_shapes_case(W, mc_shape_tool_specs(MC_WP_TOOLS + ("bcw3", "bcw-2", "geo"), bd), ctu=ctu)
    elif kind == "phases":
        pus, tags, used = _mc_phase_case(W)
    elif kind == "edges":
        pus, tags, marks = _mc_edges_case(W, H, ctu, chroma, bd); used = 0
    elif kind == "affine":
        pus, tags, used = _mc_affine_case(W, ctu)
    elif kind == "targets":
        pus, tags, targets, used = _mc_dmvr_target_case(W)
    elif kind == "surfaces":
        pus, tags, used = _mc_surface_case(W)
    assert used <= H, (name, used, H)
    pus, ndmvr = _mc_finish(pus)
    if kind == "wp":
        wp = gen_wp(np.random.default_rng(bd), bd, pus)
    refs = _mc_refs(name, W, H, bd, bool(chroma), strides, recipe, pus, tags)
    g = A.make_geom(W, H, bd, chroma_format=chroma, ctu=ctu, strides=strides or ((W, W >> 1, W >> 1) if chroma else (W, 0, 0)))
    case = dict(name=name, g=g, W=W, H=H, bd=bd, ctu=ctu, chroma=chroma, strides=(g.stride[0], g.stride[1], g.stride[2]), pus=pus, ndmvr=ndmvr, refs=refs,
                tags=tags, marks=marks, targets=targets, wp=wp)
    _mc_sweep_cache[name] = case
    return case


# ---- K3: decisions, the grid rule of the flat pass and the designed deblocking sweep (tests/test_k3_*.py)
LF_TC = (0,) * 18 + (3, 4, 4, 4, 4, 5, 5, 5, 5, 7, 7, 8, 9, 10, 10, 11, 13, 14, 15, 17, 19, 21, 24, 25, 29, 33, 36, 41, 45, 51, 57, 64, 71, 80, 89, 100, 112,
                     125, 141, 157, 177, 198, 222, 250, 280, 314, 352, 395)              # H.266 Table 43, tC'
LF_BETA = (0,) * 16 + tuple(range(6, 19)) + tuple(range(20, 89, 2))                      # H.266 Table 43, beta'
assert len(LF_TC) == 66 and len(LF_BETA) == 64


def lf_tc(idx, bd):
    return (LF_TC[idx] + (1 << (9 - bd))) >> (10 - bd) if bd < 10 else LF_TC[idx] << (bd - 10)


def lf_beta(idx, bd):
    return LF_BETA[idx] << (bd - 8)


def _clip(lo, hi, v):
    return lo if v < lo else hi if v > hi else v


def _lf_line(plane, x, y, d, line, n):
    """The samples across an edge on one line, counted from the edge: (p[0..n-1], q[0..n-1]); samples outside the array read as 0."""
    h, w = plane.shape
    at = lambda r, c: int(plane[r, c]) if 0 <= r < h and 0 <= c < w else 0
    if d == 0: return [at(y + line, x - 1 - k) for k in range(n)], [at(y + line, x + k) for k in range(n)]
    return [at(y - 1 - k, x + line) for k in range(n)], [at(y + k, x + line) for k in range(n)]


def _lf_at(x, y, d, line, side, k):
    """(row, column) of the k-th sample of the P (side 0) or Q (side 1) side of one line."""
    o = -1 - k if side == 0 else k
    return (y + line, x + o) if d == 0 else (y + o, x + line)


def _lf_strong(p, q, d, beta, tc, largeP, largeQ, maxP, maxQ, ctb=False):
    """xUseStrongFiltering (LoopFilter.cpp:1410) on one line: (decision, sp3 + sq3 as compared)."""
    ok = d < (beta >> 2) and abs(p[0] - q[0]) < ((tc * 5 + 1) >> 1)
    sp, sq = abs(p[1] - p[0]) if ctb else abs(p[3] - p[0]), abs(q[3] - q[0])
    if largeP or largeQ:
        if largeP:
            if maxP == 7: sp += abs(p[4] - p[5] - p[6] + p[7])
            sp = (sp + abs(p[3] - p[maxP]) + 1) >> 1
        if largeQ:
            if maxQ == 7: sq += abs(q[4] - q[5] - q[6] + q[7])
            sq = (sq + abs(q[maxQ] - q[3]) + 1) >> 1
        return ok and sp + sq < (beta * 3 >> 5) and d < (beta >> 4), sp + sq
    return ok and sp + sq < (beta >> 3), sp + sq


def _lf_luma(P, x, y, d, e, sl, seq, bd, ctu):
    """xEdgeFilterLuma's decisions (LoopFilter.cpp:1463) for one 4-line segment."""
    bs, qp, pmax = int(e["bs"]) & 3, int(e["qp"][0]), (1 << bd) - 1
    if seq is not None and seq.ladfEnabled:                    # deriveLADFShift :1363
        (p0, q0), (p3, q3) = _lf_line(P, x, y, d, 0, 1), _lf_line(P, x, y, d, 3, 1)
        lvl, shift = (q0[0] + q3[0] + p0[0] + p3[0]) >> 2, seq.ladfQpOffset[0]
        for k in range(1, seq.ladfNumIntervals):
            if lvl > seq.ladfIntervalLowerBound[k]: shift = seq.ladfQpOffset[k]
            else: break
        qp += shift
    maxP, maxQ = (int(e["len"]) >> 4) & 7, int(e["len"]) & 7
    largeP, largeQ = maxP > 3 and not (d == 1 and y % ctu == 0), maxQ > 3
    itc, ib = _clip(0, 65, qp + 2 * (bs - 1) + 2 * int(sl["tc"][0])), _clip(0, 63, qp + 2 * int(sl["beta"][0]))
    tc, beta = lf_tc(itc, bd), lf_beta(ib, bd)
    L = [_lf_line(P, x, y, d, l, 8) for l in range(4)]
    dp = [abs(p[2] - 2 * p[1] + p[0]) for p, q in L]; dq = [abs(q[0] - 2 * q[1] + q[2]) for p, q in L]
    Q = dict(qp=qp, itc=itc, ib=ib, tc=tc, beta=beta, beta2=beta >> 2, beta3=beta >> 3, beta4=beta >> 4, beta35=beta * 3 >> 5, tc25=(tc * 5 + 1) >> 1,
             sideThr=(beta + (beta >> 1)) >> 3, thrCut=tc * 10, dsum=dp[0] + dq[0] + dp[3] + dq[3], pq_a=abs(L[0][0][0] - L[0][1][0]), pq_b=abs(L[3][0][0] - L[3][1][0]))
    side = lambda n, m: {(l, 0, k) for l in range(4) for k in range(n)} | {(l, 1, k) for l in range(4) for k in range(m)}
    if largeP or largeQ:
        dL = [(((dp[l] + abs(L[l][0][5] - 2 * L[l][0][4] + L[l][0][3]) + 1) >> 1) if largeP else dp[l]) +
              (((dq[l] + abs(L[l][1][3] - 2 * L[l][1][4] + L[l][1][5]) + 1) >> 1) if largeQ else dq[l]) for l in (0, 3)]
        sa, sb = (_lf_strong(*L[l], 2 * dL[i], beta, tc, largeP, largeQ, maxP, maxQ) for i, l in enumerate((0, 3)))
        Q.update(dsumL=dL[0] + dL[1], d2L_a=2 * dL[0], d2L_b=2 * dL[1], sL_a=sa[1], sL_b=sb[1])
        if Q["dsumL"] < beta and sa[0] and sb[0]:
            nP, nQ = maxP if largeP else 3, maxQ if largeQ else 3
            return f"long{nP}{nQ}", side(nP, nQ), Q
    if Q["dsum"] >= beta: return "none", set(), Q
    fP = fQ = sw = False
    if maxP > 1 and maxQ > 1: fP, fQ = dp[0] + dp[3] < Q["sideThr"], dq[0] + dq[3] < Q["sideThr"]
    Q.update(pside=dp[0] + dp[3], qside=dq[0] + dq[3])
    if maxP > 2 and maxQ > 2:
        sa, sb = (_lf_strong(*L[l], 2 * (dp[l] + dq[l]), beta, tc, False, False, 7, 7) for l in (0, 3))
        Q.update(d2_a=2 * (dp[0] + dq[0]), d2_b=2 * (dp[3] + dq[3]), s_a=sa[1], s_b=sb[1])
        sw = sa[0] and sb[0]
    if sw: return "strong", side(3, 3), Q
    writes, deltas, clip01 = set(), [], False
    for l, (p, q) in enumerate(L):
        delta = (9 * (q[0] - p[0]) - 3 * (q[1] - p[1]) + 8) >> 4
        deltas.append(delta)
        if abs(delta) >= Q["thrCut"]: continue
        dc, t2 = _clip(-tc, tc, delta), tc >> 1
        new = [p[0] + dc, q[0] - dc] + ([p[1] + _clip(-t2, t2, (((p[2] + p[0] + 1) >> 1) - p[1] + dc) >> 1)] if fP else []) + \
              ([q[1] + _clip(-t2, t2, (((q[2] + q[0] + 1) >> 1) - q[1] - dc) >> 1)] if fQ else [])
        clip01 |= any(v < 0 or v > pmax for v in new)
        writes |= {(l, 0, 0), (l, 1, 0)} | ({(l, 0, 1)} if fP else set()) | ({(l, 1, 1)} if fQ else set())
    Q.update(adelta_a=abs(deltas[0]), adelta_b=abs(deltas[3]), clip01=clip01)
    return ("weak_cut" if not writes else f"weak{int(fP)}{int(fQ)}"), writes, Q


def _lf_chroma(P, cx, cy, d, e, sl, c, bd, ctu):
    """xEdgeFilterChroma's decisions (LoopFilter.cpp:1619) for one 2-line segment of component c (4:2:0)."""
    bs, large = (int(e["bs"]) >> (2 * c)) & 3, (int(e["flags"]) >> 5) & 1
    ctb = d == 1 and cy % (ctu >> 1) == 0
    sfx = "_ctb" if ctb else ""
    if not (bs == 2 or (large and bs == 1)): return "none" + sfx, set(), {}
    qp = int(e["qp"][c])
    itc = _clip(0, 65, qp + 2 * (bs - 1) + 2 * int(sl["tc"][c])); tc = lf_tc(itc, bd)
    Q = dict(qp=qp, itc=itc, tc=tc, tc25=(tc * 5 + 1) >> 1)
    weak = {(l, s, 0) for l in range(2) for s in range(2)}
    if not large: return "chroma_weak_small" + sfx, weak, Q
    ib = _clip(0, 63, qp + 2 * int(sl["beta"][c])); beta = lf_beta(ib, bd)
    L = [_lf_line(P, cx, cy, d, l, 4) for l in range(2)]
    dl = [(abs(p[0] - p[1]) if ctb else abs(p[2] - 2 * p[1] + p[0])) + abs(q[0] - 2 * q[1] + q[2]) for p, q in L]
    Q.update(ib=ib, beta=beta, beta2=beta >> 2, beta3=beta >> 3, dsum=dl[0] + dl[1], d2_a=2 * dl[0], d2_b=2 * dl[1],
             pq_a=abs(L[0][0][0] - L[0][1][0]), pq_b=abs(L[1][0][0] - L[1][1][0]))
    if Q["dsum"] >= beta: return "chroma_weak_d" + sfx, weak, Q
    sa, sb = (_lf_strong(*L[l], 2 * dl[l], beta, tc, False, False, 7, 7, ctb) for l in range(2))
    Q.update(s_a=sa[1], s_b=sb[1])
    if sa[0] and sb[0]:
        return "chroma_strong" + sfx, {(l, 0, k) for l in range(2) for k in range(1 if ctb else 3)} | {(l, 1, k) for l in range(2) for k in range(3)}, Q
    return "chroma_weak" + sfx, weak, Q


def lf_decisions(planes, grid, d, g, slices, seq=None, ctu_slice=None):
    """The decisions of xEdgeFilterLuma / xEdgeFilterChroma (not the filters) for every segment of one direction's grid (d: 0 lfV, 1 lfH) on `planes`,
    the picture that direction starts from (for lfH: the output of the vertical pass).  Returns one dict per segment: dir, comp, x / y (the first Q
    sample, in the component's plane), tag (none, weak00..weak11, weak_cut, strong, long<P><Q>, chroma_weak_small / _d / chroma_weak / chroma_strong,
    + _ctb at a chroma CTB row, off in a slice with deblocking disabled), writes (the (row, column) samples the decision may change) and q (the
    quantities and thresholds it compared)."""
    out = []
    bd, ctu = g.bitDepth, g.ctuSize
    ctus_w = (g.width + ctu - 1) // ctu
    ys, xs = np.nonzero(grid["bs"] & 0x3f)
    for y4, x4 in zip(ys.tolist(), xs.tolist()):
        e, x, y = grid[y4, x4], 4 * x4, 4 * y4
        sl = slices[int(ctu_slice[(y // ctu) * ctus_w + x // ctu]) if ctu_slice is not None else 0]
        segs = []
        if int(e["bs"]) & 3: segs.append((0, x, y, 4))
        if g.chromaFormat == 1 and int(e["bs"]) >> 2 and (x if d == 0 else y) % 16 == 0:
            segs += [(c, x >> 1, y >> 1, 2) for c in (1, 2) if (int(e["bs"]) >> (2 * c)) & 3]
        for c, cx, cy, n in segs:
            if sl["disable"]: tag, w, q = "off", set(), {}
            elif c == 0: tag, w, q = _lf_luma(planes[0], x, y, d, e, sl, seq, bd, ctu)
            else: tag, w, q = _lf_chroma(planes[c], cx, cy, d, e, sl, c, bd, ctu)
            out.append(dict(dir=d, comp=c, x=cx, y=cy, tag=tag, q=q, writes={_lf_at(cx, cy, d, l, s, k) for l, s, k in w}))
    return out


def _lf_side(v, d=0, s=0, dx=0, e=0, a1=0):
    """Eight samples of one side of an edge, nearest first, around level v: |x2 - 2 x1 + x0| = d, |x3 - x0| = s, |x5 - 2 x4 + x3| = dx, and at length 7
    |x4 - x5 - x6 + x7| = e with x7 = x3 (length 5: |x3 - x5| = dx); a1 = x1 - x0 (the chroma CTB form's |p1 - p0|)."""
    return [v, v + a1, v + d + 2 * a1, v + s, v + s, v + s + dx, v + s - dx - e, v + s]


class _LfCanvas:
    """A picture being laid out for the deblocking sweep: planes at mid grey, empty grids, and the designed segments placed so far."""
    def __init__(self, W, H, bd, ctu, chroma=1, strides=None, fill=-7):
        self.g = abi.make_geom(W, H, bd, chroma_format=chroma, ctu=ctu, strides=strides or ((W, W >> 1, W >> 1) if chroma else (W, 0, 0)))
        self.W, self.H, self.bd, self.ctu, self.chroma = W, H, bd, ctu, chroma
        mid = 1 << (bd - 1)
        self.planes = [None, None, None]
        for c in range(3 if chroma else 1):
            w, h = (W, H) if c == 0 else (W >> 1, H >> 1)
            self.planes[c] = np.full((h, self.g.stride[c]), fill, np.int16); self.planes[c][:, :w] = mid
        self.lf = [np.zeros((H // 4, W // 4), LF_DTYPE) for _ in range(2)]
        self.segs = []

    def put(self, spec, d, x, y):
        """Writes a designed segment across the edge at luma (x, y): spec = dict(tag, comp (0 luma, 'c' both chroma), lens, bs, qp, large, lines,
        probes) where lines are the (p, q) sample lists of each line (4 luma, 2 chroma)."""
        e = self.lf[d][y // 4, x // 4]
        comps = (0,) if spec.get("comp", 0) == 0 else (1, 2)
        bs = spec.get("bs", 2)
        e["bs"] = bs if comps == (0,) else (bs << 2) | (bs << 4)
        e["len"] = 128 + (spec.get("lens", (3, 3))[0] << 4) + spec.get("lens", (3, 3))[1]
        e["flags"] = 32 if spec.get("large") else 0
        e["qp"] = (spec.get("qp", 37),) * 3
        for c in comps:
            cx, cy = (x, y) if c == 0 else (x >> 1, y >> 1)
            for l, (p, q) in enumerate(spec["lines"]):
                for s, vals in ((0, p), (1, q)):
                    for k, v in enumerate(vals[:8 if c == 0 else 4]): self.planes[c][_lf_at(cx, cy, d, l, s, k)] = v    # a chroma slot holds 4 per side
            self.segs.append(dict(dir=d, comp=c, x=cx, y=cy, tag=spec["tag"], probes=spec.get("probes", [])))

    def case(self, name, slices=None, ctu_slice=None, seq=None, classify=True):
        return dict(name=name, g=self.g, W=self.W, H=self.H, bd=self.bd, ctu=self.ctu, chroma=self.chroma, strides=tuple(self.g.stride),
                    planes=self.planes, lfV=np.ascontiguousarray(self.lf[0]), lfH=np.ascontiguousarray(self.lf[1]),
                    slices=np.zeros(1, LFSLICE_DTYPE) if slices is None else slices, ctuSlice=ctu_slice, seq=seq or abi.LfSeq(), segs=self.segs, classify=classify)


def _lf_spec(tag, l0, l3=None, v=512, lens=(3, 3), bs=2, qp=37, probes=(), nlines=4, **kw):
    """A designed segment: line 0 (and the lines up to the last) shaped by l0 = dict(t, dp, dq, sp, sq, dpx, dqx, ep, eq, ap, aq) around level v (Q side at
    v + t); the last line (3 luma, 1 chroma) by l0 updated with l3."""
    def line(k):
        t = k.get("t", 20)
        return (_lf_side(v, k.get("dp", 0), k.get("sp", 0), k.get("dpx", 0), k.get("ep", 0), k.get("ap", 0)),
                _lf_side(v + t, k.get("dq", 0), k.get("sq", 0), k.get("dqx", 0), k.get("eq", 0), k.get("aq", 0)))
    last = dict(l0, **(l3 or {}))
    return dict(tag=tag, lens=lens, bs=bs, qp=qp, probes=list(probes), lines=[line(l0)] * (nlines - 1) + [line(last)], **kw)


def lf_luma_specs():
    """The designed luma segments (10 bit): thresholds of every decision of xEdgeFilterLuma on both sides.  qp 37 / Bs 2: beta 144, tc 21 (beta>>2 36,
    beta>>3 18, side threshold 27, (5 tc + 1)>>1 53); qp 39: beta 160, tc 25 (beta>>4 10, 3 beta>>5 15, 63); qp 18 / Bs 1: beta 32, tc 3 (thrCut 30)."""
    S = []
    # no filter at d0 + d3 == beta, weak below
    S += [_lf_spec("none", dict(dp=5, dq=66), dict(dq=68), probes=[("dsum", "beta", 0)]),
          _lf_spec("weak10", dict(dp=5, dq=66), dict(dq=67), probes=[("dsum", "beta", -1)])]
    # |delta| at thrCut and one below (flat sides: delta = (6 t + 8) >> 4)
    S += [_lf_spec("weak_cut", dict(t=79), qp=18, bs=1, probes=[("adelta_a", "thrCut", 0)]),
          _lf_spec("weak11", dict(t=76), qp=18, bs=1, probes=[("adelta_a", "thrCut", -1)])]
    # the side taps at the side threshold and one below (sp3 20 keeps strong off)
    for fP in (0, 1):
        for fQ in (0, 1):
            S.append(_lf_spec(f"weak{fP}{fQ}", dict(t=30, sp=20, dp=13, dq=13), dict(dp=14 - fP, dq=14 - fQ),
                              probes=[("pside", "sideThr", -fP), ("qside", "sideThr", -fQ)]))
    # delta clipped to +-tc (and exactly tc)
    S += [_lf_spec("weak11", dict(t=60), probes=[("adelta_a", "tc", 2)]), _lf_spec("weak11", dict(t=-60), v=600, probes=[("adelta_a", "tc", 1)]),
          _lf_spec("weak11", dict(t=56), probes=[("adelta_a", "tc", 0)]), _lf_spec("weak11", dict(t=53), probes=[("adelta_a", "tc", -1)])]
    # normal strong, and each of its conditions failing alone on line 0 only and on line 3 only
    base = dict(dp=2, dq=2, t=20)
    S.append(_lf_spec("strong", base, probes=[("d2_a", "beta2", -28), ("pq_a", "tc25", -33), ("s_a", "beta3", -18)]))
    for ln, key in ((0, "a"), (3, "b")):
        for cond, fail, ok, q, thr, okoff in (("d", dict(dp=9, dq=9), dict(dp=8, dq=9), "d2", "beta2", -2), ("pq", dict(t=53), dict(t=52), "pq", "tc25", -1),
                                              ("s", dict(sp=18), dict(sp=17), "s", "beta3", -1)):
            for tag, ch, off in (("weak11", fail, 0), ("strong", ok, okoff)):
                l0, l3 = (dict(base, **ch), dict(base)) if ln == 0 else (base, ch)
                S.append(_lf_spec(tag, l0, l3, probes=[(f"{q}_{key}", thr, off)]))
    # every long pair, and each long condition failing alone on line 0 (the segment then takes the normal decision)
    for P, Q in ((5, 3), (3, 5), (5, 5), (5, 7), (7, 5), (7, 3), (3, 7), (7, 7)):
        big = "p" if P > 3 else "q"
        S.append(_lf_spec(f"long{P}{Q}", dict(t=20), lens=(P, Q), qp=39, probes=[("d2L_a", "beta4", -10), ("sL_a", "beta35", -15), ("pq_a", "tc25", -43)]))
        for fail, ok, q, thr, off, ftag in ((dict(**{f"d{big}x": 9}), dict(**{f"d{big}x": 7}), "d2L_a", "beta4", -2, "strong"),
                                            (dict(**{f"s{big}": 29}), dict(**{f"s{big}": 27}), "sL_a", "beta35", -1, "weak11"),
                                            (dict(t=63), dict(t=62), "pq_a", "tc25", -1, "weak11")):
            S.append(_lf_spec(ftag, dict({"t": 20}, **fail), dict(t=20), lens=(P, Q), qp=39, probes=[(q, thr, 0)]))
            S.append(_lf_spec(f"long{P}{Q}", dict({"t": 20}, **ok), dict(t=20), lens=(P, Q), qp=39, probes=[(q, thr, off)]))
    # lengths 1/1 and 2/2: strong is off on content that would take it, the side taps follow the length
    S += [_lf_spec("weak00", base, lens=(1, 1)), _lf_spec("weak11", base, lens=(2, 2)), _lf_spec("weak01", dict(base, dp=13), dict(dp=14), lens=(2, 2))]
    return S


def lf_chroma_specs(ctb):
    """The designed chroma segments (10 bit, qp 37: beta 144, tc 21 at Bs 2 / 17 at Bs 1): Bs 1 / 2 x large 0 / 1, and a large edge's strong filter
    failing one condition at a time; ctb: the forms of a horizontal CTB boundary (P side of two rows)."""
    sfx, C = ("_ctb" if ctb else ""), []
    sp = lambda k: dict(ap=k) if ctb else dict(sp=k)          # what sp3 measures: |p1 - p0| at a CTB boundary, else |p3 - p0|
    spec = lambda tag, l0, l1=None, **kw: _lf_spec(tag + sfx, l0, l1, nlines=2, comp="c", **kw)
    C += [spec("none", dict(t=20), bs=1), spec("chroma_weak_small", dict(t=20)), spec("chroma_strong", dict(t=20), bs=1, large=1),
          spec("chroma_strong", dict(t=20), large=1, probes=[("pq_a", "tc25", -33)]),
          spec("chroma_weak_d", dict(dq=72), large=1, probes=[("dsum", "beta", 0)]), spec("chroma_weak", dict(dq=72), dict(dq=71), large=1, probes=[("dsum", "beta", -1)])]
    for ln, key in ((0, "a"), (1, "b")):
        for fail, ok, q, thr, off in ((dict(dq=18), dict(dq=17), "d2", "beta2", -2), (dict(t=53), dict(t=52), "pq", "tc25", -1), (dict(sq=18), dict(sq=17), "s", "beta3", -1)):
            for tag, ch, o in (("chroma_weak", fail, 0), ("chroma_strong", ok, off)):
                l0, l1 = (dict({"t": 20}, **ch), dict(t=20)) if ln == 0 else (dict(t=20), dict({"t": 20}, **ch))
                C.append(spec(tag, l0, l1, large=1, probes=[(f"{q}_{key}", thr, o)]))
    C.append(spec("chroma_weak", dict({"t": 20}, **sp(18)), large=1, probes=[("s_a", "beta3", 0)]))
    return C


def _lf_layout(cv, vspecs, hspecs, y0=0):
    """Places segments: vertical edges in 32 x 4 luma slots from row y0 (edge at +16), horizontal ones in 4 x 16 slots below (edge at +8, on the 16-row
    chroma grid); a horizontal spec with ctb=True goes to a CTU row, the others avoid CTU rows.  Returns the rows used."""
    per = cv.W // 32
    for i, s in enumerate(vspecs): cv.put(s, 0, 32 * (i % per) + 16, y0 + 4 * (i // per))
    y = y0 + 4 * ((len(vspecs) + per - 1) // per)
    ye = (y + 8 + 15) // 16 * 16
    todo = {True: [s for s in hspecs if s.get("ctb")], False: [s for s in hspecs if not s.get("ctb")]}
    end = y
    while todo[True] or todo[False]:
        row = todo[ye % cv.ctu == 0]
        for i in range(min(len(row), cv.W // 4)): cv.put(row.pop(0), 1, 4 * i, ye)
        end, ye = ye + 8, ye + 16
    return end


def _lf_blocks(extent, pattern):
    """Blocks along one axis: `pattern` (sizes; ('sb', n): a CU of n coded in 8-sample sub-blocks) repeated until the extent is covered, the last block
    cut to fit.  Returns the edges as (position, P length, Q length), derived as xSetMaxFilterLengthPQFromTransformSizes (LoopFilter.cpp:780) and
    xSetMaxFilterLengthPQForCodingSubBlocks (:707) do, and the index of the (sub-)block every sample lies in."""
    blocks, pos, i = [], 0, 0
    while pos < extent:
        it = pattern[i % len(pattern)]; i += 1
        sb, n = (True, it[1]) if isinstance(it, tuple) else (False, it)
        n = min(n, extent - pos)
        blocks.append((pos, n, sb and n >= 16)); pos += n
    edges, idx, k = [], np.zeros(extent, np.int64), 0
    for j, (b0, n, sb) in enumerate(blocks):
        if j:
            a0, an, asb = blocks[j - 1]
            P, Q = (1, 1) if min(an, n) <= 4 else (7 if an >= 32 else 3, 7 if n >= 32 else 3)
            if asb: P = min(P, 5)
            if sb: Q = min(Q, 5)
            edges.append((b0, P, Q))
        subs = range(b0, b0 + n, 8) if sb else [b0]
        for s in subs:
            if s > b0: edges.append((s, 2, 2) if s - b0 == 8 or s - b0 + 8 >= n else (s, 3, 3))
            idx[s:b0 + n] = k; k += 1
    return edges, idx


def _lf_block_case(cv, xpat, ypat, t, qp=37, chroma_bs=(2, 1)):
    """A picture of flat blocks (block (i, j) at level mid + t * ((i % 2) + (j % 3))) and the grids of their edges, every 4x4 unit of an edge with luma
    Bs 2; chroma Bs alternates between the values of chroma_bs, and the chroma 'large' flag is set where both blocks are at least 16 luma samples."""
    xe, xi = _lf_blocks(cv.W, xpat); ye, yi = _lf_blocks(cv.H, ypat)
    mid = 1 << (cv.bd - 1)
    Y = mid + t * ((xi[None, :] % 2) + (yi[:, None] % 3))
    cv.planes[0][:, :cv.W] = Y
    for c in (1, 2) if cv.chroma else ():
        cv.planes[c][:, :cv.W >> 1] = Y[::2, ::2] - (c - 1) * t
    size_at = lambda edges, extent: np.diff([0] + [e[0] for e in edges] + [extent])
    for d, edges, other in ((0, xe, cv.H), (1, ye, cv.W)):
        sizes = size_at(edges, cv.W if d == 0 else cv.H)
        for k, (pos, P, Q) in enumerate(edges):
            cb = chroma_bs[k % len(chroma_bs)]
            sl = (slice(None), pos // 4) if d == 0 else (pos // 4, slice(None))
            e = cv.lf[d][sl]
            e["bs"] = 2 | (cb << 2) | (cb << 4)
            e["len"] = 128 + (P << 4) + Q
            e["flags"] = 32 if min(sizes[k], sizes[k + 1]) >= 16 else 0
            e["qp"] = (qp, qp - 1, qp + 1)
    return cv


_LF_TIGHT = ([32, 4, 4, 4, 4, 8, 8, 8, 8, ("sb", 64), 32, 16, 8, 4, 4, 16, ("sb", 32), 32], [32, 8, 8, 4, 4, 8, 16, 32, ("sb", 32), 8, 8, 16, 32])


def _lf_qp_specs(bd, ladf=None):
    """Segments for one bit depth: for every Bs 1 / 2 and QP from -6 (bd - 8) to 63 (every 3rd), flat sides and a step sized so that a weak filter's delta
    is about 2 tc (clipped to tc) and strong filtering fails; QP 63 with Bs 2 (tc index clipped at 65).  ladf: (level, qp) pairs, each a segment whose
    LADF luma level is `level` exactly (P side level - k, Q side + k)."""
    S, mid, pmax = [], 1 << (bd - 1), (1 << bd) - 1
    pairs = ladf or [(None, qp) for qp in list(range(-6 * (bd - 8), 64, 3)) + [63]]
    for lvl, qp in pairs:
        for bs in (1, 2):
            tc = lf_tc(_clip(0, 65, qp + 2 * (bs - 1)), bd)
            t = _clip(2, pmax // 3, (32 * tc) // 6 + 2) // 2 * 2
            v = (lvl if lvl is not None else mid) - t // 2
            S.append(_lf_spec("any", dict(t=t), v=v, bs=bs, qp=qp))
            S.append(_lf_spec("any", dict(t=-t), v=v + t, bs=bs, qp=qp))
            S.append(_lf_spec("any", dict(t=t // 3, dp=1, dq=2), v=v, bs=bs, qp=qp))
    return S


def _lf_clip_specs(bd):
    """Content at 0 and at the largest sample value with tc at its maximum (qp 63, Bs 2): the weak filter's result leaves [0, pmax] and is clipped; large
    steps through the strong and long filters."""
    pmax, S = (1 << bd) - 1, []
    for flip in (False, True):
        f = (lambda a: [pmax - x for x in a]) if flip else (lambda a: a)
        p, q = [pmax - 95, pmax, pmax, pmax - 95, pmax - 95, pmax - 95, pmax - 95, pmax - 95], [pmax, pmax - 495, pmax - 990, pmax - 495] + [pmax - 495] * 4
        S.append(dict(tag="weak11", qp=63, lines=[(f(p), f(q))] * 4, probes=[]))
        p2 = [pmax - 300, pmax, pmax, pmax - 300] + [pmax - 300] * 4
        S.append(dict(tag="weak01", qp=63, lines=[(f(p2), f(q))] * 4, probes=[]))
    for lens, t in (((3, 3), 3000), ((7, 7), 3500), ((5, 3), 3900), ((7, 3), 2000)):
        for flip in (False, True):
            lo, hi = (0, t) if not flip else (pmax, pmax - t)
            S.append(_lf_spec("any", dict(t=hi - lo), v=lo, lens=lens, qp=63))
    return S


def _lf_ctu_specs():
    """Horizontal luma edges on CTU rows with a long P side, whose P side is run as length 3: the P side is flat for 4 rows and then steps by 40, so a
    long P side would decide or filter differently."""
    S = []
    for (P, Q), tag in (((7, 7), "long37"), ((5, 7), "long37"), ((7, 5), "long35"), ((5, 5), "long35"), ((7, 3), "strong"), ((5, 3), "strong")):
        s = _lf_spec(tag, dict(t=20), lens=(P, Q), qp=39, ctb=True)
        for p, q in s["lines"]: p[4:] = [x + 40 for x in p[4:]]
        S.append(s)
    return S


def _lf_slices(n, disable_every=5):
    sl = np.zeros(n, LFSLICE_DTYPE)
    for i in range(n):
        sl[i]["beta"] = [((i + 5 * c) % 25) - 12 for c in range(3)]
        sl[i]["tc"] = [((7 * i + 3 * c) % 25) - 12 for c in range(3)]
        sl[i]["disable"] = i % disable_every == 3
    return sl


def _lf_ladf(bd):
    """Five LADF intervals with shifts that take low QPs below 0, and (level, qp) pairs on each lower bound and one above it."""
    s = abi.LfSeq(); s.ladfEnabled, s.ladfNumIntervals = 1, 5
    sc = 1 << (bd - 8)
    bounds, offs = [0, 40 * sc, 90 * sc, 140 * sc, 200 * sc], [-3, 4, -12, 7, -30]
    for k in range(5): s.ladfQpOffset[k] = offs[k]; s.ladfIntervalLowerBound[k] = bounds[k]
    pairs = [(lvl, qp) for b in bounds[1:] for lvl in (b, b + 1) for qp in (4, 30, 45)] + [(10 * sc, 20), (250 * sc, 20)]
    return s, pairs


def _lf_case(name):
    kind, *a = LF_SWEEP_CASES[name]
    if kind == "luma":
        specs = lf_luma_specs()
        cv = _LfCanvas(1024, 512, 10, 128)
        used = _lf_layout(cv, specs, [dict(s) for s in specs])
        assert used <= cv.H, used
        return cv.case(name)
    if kind == "chroma":
        ctu, W, H = a
        cv = _LfCanvas(W, H, 10, ctu)
        hs = lf_chroma_specs(False) + [dict(s, ctb=True) for s in lf_chroma_specs(True)]
        assert _lf_layout(cv, lf_chroma_specs(False), hs) <= H
        return cv.case(name)
    if kind == "qp":
        bd, ladf = a
        seq, pairs = _lf_ladf(bd) if ladf else (None, None)
        specs = _lf_qp_specs(bd, pairs)
        cv = _LfCanvas(512, 512 if not ladf else 256, bd, 32)
        assert _lf_layout(cv, specs, [dict(s) for s in specs]) <= cv.H
        # slices by CTU column: offsets 0, +12, -12 and mixed, for every component
        sl = np.zeros(4, LFSLICE_DTYPE)
        sl["beta"][1], sl["tc"][1] = 12, 12
        sl["beta"][2], sl["tc"][2] = -12, -12
        sl["beta"][3], sl["tc"][3] = (12, -12, 6), (-12, 12, -6)
        nw, nh = cv.W // 32, cv.H // 32
        cs = np.array([(i % nw) % 4 if not ladf else 0 for i in range(nw * nh)], np.uint8)
        return cv.case(name, slices=sl if not ladf else None, ctu_slice=cs, seq=seq)
    if kind == "clip":
        cv = _LfCanvas(256, 128, 12, 128)
        specs = _lf_clip_specs(12)
        assert _lf_layout(cv, specs, [dict(s) for s in specs]) <= cv.H
        return cv.case(name)
    if kind == "blocks":
        W, H, bd, ctu, chroma, strides, xpat, ypat, t, nsl = a
        cv = _lf_block_case(_LfCanvas(W, H, bd, ctu, chroma, strides), xpat, ypat, t)
        if nsl <= 1: return cv.case(name, classify=W * H <= 1 << 20)
        nctu = ((W + ctu - 1) // ctu) * ((H + ctu - 1) // ctu)
        cs = np.array([(37 * i) % nsl for i in range(nctu)], np.uint8)
        return cv.case(name, slices=_lf_slices(nsl), ctu_slice=cs)
    if kind == "ctu":
        ctu, W, H = a
        cv = _LfCanvas(W, H, 10, ctu)
        specs = _lf_ctu_specs()
        _lf_layout(cv, [], specs * (W // 4 // len(specs)), y0=ctu - 16)
        return cv.case(name)
    raise KeyError(name)


LF_SWEEP_CASES = {
    "luma_decisions_10bit": ("luma",),
    "chroma_decisions_10bit": ("chroma", 128, 256, 320),
    "chroma_ctb_ctu32": ("chroma", 32, 256, 320),
    "chroma_ctb_ctu64": ("chroma", 64, 256, 320),
    "qp_extremes_8bit": ("qp", 8, False), "qp_extremes_9bit": ("qp", 9, False), "qp_extremes_10bit": ("qp", 10, False), "qp_extremes_12bit": ("qp", 12, False),
    "qp_ladf_10bit": ("qp", 10, True), "qp_ladf_12bit": ("qp", 12, True),
    "clipping_12bit": ("clip",),
    "tight_spacing": ("blocks", 512, 256, 10, 128, 1, None, *_LF_TIGHT, 12, 1),
    "ctu_rows_ctu32": ("ctu", 32, 256, 64), "ctu_rows_ctu64": ("ctu", 64, 256, 128), "ctu_rows_ctu128": ("ctu", 128, 256, 256),
    "ctu_edges_ctu32_200x136": ("blocks", 200, 136, 10, 32, 1, None, [8, 8, 16, 32, 4, 4, 8, 16], [32, 16, 8, 8, 32, ("sb", 32)], 12, 1),
    "ctu_edges_ctu64_416x240": ("blocks", 416, 240, 10, 64, 1, None, [32, 32, 16, 16, 32, ("sb", 64), 64], [64, 32, 16, 16, ("sb", 32), 32], 12, 1),
    "ctu_edges_ctu128_1928x1080": ("blocks", 1928, 1080, 10, 128, 1, None, [64, 64, 32, 32, 16, 16, 8, 8, 4, 4, 8, 8, 16, 32, ("sb", 64), 32, 32],
                                   [128, 64, 32, 32, 64, 16, 16, 32], 12, 1),
    "slices_64": ("blocks", 512, 128, 10, 32, 1, None, *_LF_TIGHT, 12, 64),
    "geometry_400_8bit": ("blocks", 256, 128, 8, 64, 0, None, *_LF_TIGHT, 4, 1),
    "geometry_400_stride": ("blocks", 256, 128, 10, 128, 0, (264, 0, 0), *_LF_TIGHT, 12, 1),
    "geometry_strides": ("blocks", 256, 128, 10, 128, 1, (263, 133, 140), *_LF_TIGHT, 12, 1),
    "uhd_3840x2160": ("blocks", 3840, 2160, 10, 128, 1, None, *_LF_TIGHT, 12, 1),
}

_lf_sweep_cache = {}


def lf_sweep(name):
    """One case of the designed K3 sweep (LF_SWEEP_CASES) as a dict: geometry (g, W, H, bd, ctu, chroma, strides), the planes (stride padding holds -7),
    the grids lfV / lfH, ctuSlice (None: every CTU in slice 0), the slice table, the LfSeq, and segs: the designed segments (dir, comp, x, y in the
    component's plane, the tag the decision is designed to take ('any': content for the comparisons only) and probes (quantity, threshold, offset):
    lf_decisions' q[quantity] - q[threshold] == offset).  classify: whether the picture is small enough to classify every segment in Python."""
    if name not in _lf_sweep_cache: _lf_sweep_cache[name] = _lf_case(name)
    c = _lf_sweep_cache[name]
    return dict(c, planes=[None if p is None else p.copy() for p in c["planes"]])


# ---- K4 / K5: the designed SAO and ALF sweep ----------------------------------------------------------------------------------------------------------
def sao_max_offset(bd):
    """The largest legal SAO offset magnitude: (1 << (min(bd, 10) - 5)) - 1, scaled by 1 << (bd - min(bd, 10)): 7, 15, 31, 31, 62, 124 at 8..12 bit."""
    b = min(bd, 10)
    return ((1 << (b - 5)) - 1) << (bd - b)


def alf_clip_values(bd):
    """m_alfClippVls: the clipping value of clip index 0..3."""
    return [1 << bd, 1 << (bd - 3), 1 << (bd - 5), 1 << (bd - 7)]


def _k45_planes(W, H, chroma, strides, content):
    """Planes (stride padding holds -7) with content(c, w, h) -> (h, w) samples."""
    out = []
    for c in range(3 if chroma else 1):
        w, h = (W, H) if c == 0 else (W // 2, H // 2)
        p = np.full((h, strides[c] if strides else w), -7, np.int16)
        p[:, :w] = content(c, w, h)
        out.append(p)
    return out


def alf_class_sums(plane, bd, ctu):
    """Restates the ALF luma classification only (deriveClassificationBlk, AdaptiveLoopFilter.cpp:969) for every 4x4 block of `plane` (h, w), picture
    borders replicated as prepareCTU does, the CTU virtual boundary at vbPos = ctu - 4.  Returns (h/4, w/4) arrays sV, sH, sD0, sD1, act, cls, tr, vb
    (the block lies at vbPos - 4 or vbPos: x96 activity and one row pair skipped) and cmp / nz, (5, h/4, w/4): the sign of sV - sH, sD0 - sD1,
    d1*hv0 - hv1*d0, hvd1 - 2*hvd0, 2*hvd1 - 9*hvd0 and whether the larger side of that comparison is nonzero."""
    h, w = plane.shape
    P = np.pad(plane.astype(np.int64), 4, mode="edge")
    vbPos = ctu - 4
    by, bx = np.arange(h // 4) * 4, np.arange(w // 4) * 4
    above, below = by % ctu == vbPos - 4, by % ctu == vbPos

    def p(yy, xx):
        return P[yy[:, None] + 4, xx[None, :] + 4]
    S = np.zeros((4, len(by), len(bx)), np.int64)
    for r in range(4):
        Y = by - 2 + 2 * r
        up = np.where((Y > 0) & (Y % ctu == vbPos), 0, -1)
        dn2 = np.where((Y > 0) & (Y % ctu == vbPos - 2), 1, 2)
        keep = ~((above & (r == 3)) | (below & (r == 0)))[:, None]
        for c in range(4):
            X = bx - 2 + 2 * c
            a, b = 2 * p(Y, X), 2 * p(Y + 1, X + 1)
            S[0] += keep * (abs(a - p(Y + up, X) - p(Y + 1, X)) + abs(b - p(Y, X + 1) - p(Y + dn2, X + 1)))
            S[1] += keep * (abs(a - p(Y, X + 1) - p(Y, X - 1)) + abs(b - p(Y + 1, X + 2) - p(Y + 1, X)))
            S[2] += keep * (abs(a - p(Y + up, X - 1) - p(Y + 1, X + 1)) + abs(b - p(Y, X) - p(Y + dn2, X + 2)))
            S[3] += keep * (abs(a - p(Y + 1, X - 1) - p(Y + up, X + 1)) + abs(b - p(Y + dn2, X) - p(Y, X + 2)))
    sV, sH, sD0, sD1 = S
    vb = np.broadcast_to((above | below)[:, None], sV.shape)
    act = np.clip(((sV + sH) * np.where(vb, 96, 64)) >> (bd + 4), 0, 15)
    hvgt, dgt = sV > sH, sD0 > sD1
    hv1, hv0, dirHV = np.where(hvgt, sV, sH), np.where(hvgt, sH, sV), np.where(hvgt, 1, 3)
    d1, d0, dirD = np.where(dgt, sD0, sD1), np.where(dgt, sD1, sD0), np.where(dgt, 0, 2)
    useD = d1 * hv0 > hv1 * d0
    hvd1, hvd0 = np.where(useD, d1, hv1), np.where(useD, d0, hv0)
    main, sec = np.where(useD, dirD, dirHV), np.where(useD, dirHV, dirD)
    strength = np.where(2 * hvd1 > 9 * hvd0, 2, np.where(hvd1 > 2 * hvd0, 1, 0))
    cls = np.array([0, 1, 2, 2, 2, 2, 2, 3, 3, 3, 3, 3, 3, 3, 3, 4])[act] + np.where(strength > 0, ((main & 1) * 2 + strength) * 5, 0)
    tr = np.array([0, 1, 0, 2, 2, 3, 1, 3])[main * 2 + (sec >> 1)]
    cmp = np.sign(np.stack([sV - sH, sD0 - sD1, d1 * hv0 - hv1 * d0, hvd1 - 2 * hvd0, 2 * hvd1 - 9 * hvd0]))
    nz = np.stack([sV > 0, sD0 > 0, d1 * hv0 > 0, hvd1 > 0, hvd1 > 0])
    return dict(sV=sV, sH=sH, sD0=sD0, sD1=sD1, act=act, cls=cls, tr=tr, vb=vb, cmp=cmp, nz=nz)


def alf_class_keys(cs, mask=None):
    """The coverage keys of classified blocks (alf_class_sums): ('ct', class, transpose), ('act', a), ('cmp', k, sign) (sign 0 only with nonzero sides)
    and ('vb', act > 0) for the blocks at the virtual boundary rows."""
    m = np.ones(cs["cls"].shape, bool) if mask is None else mask
    keys = {("ct", int(c), int(t)) for c, t in zip(cs["cls"][m], cs["tr"][m])} | {("act", int(a)) for a in np.unique(cs["act"][m])}
    for k in range(5):
        s, z = cs["cmp"][k][m], cs["nz"][k][m]
        keys |= {("cmp", k, int(v)) for v in np.unique(s[(s != 0) | z])}
    keys |= {("vb", bool(a > 0)) for a in np.unique(cs["act"][m & cs["vb"]])}
    return keys


def _alf_cell_pool(bd, n, seed):
    """n 12x12 cells of mixed stripe / diagonal / checkerboard texture at amplitudes from pmax/2 down to nothing (ties between the Laplacian sums
    are frequent at small amplitudes), plus step cells whose neighbour differences sit at every clipping value -1, +0, +1."""
    rng = np.random.default_rng(seed)
    pmax = (1 << bd) - 1
    yy, xx = np.mgrid[0:12, 0:12]
    pats = np.stack([(-1.0) ** yy, (-1.0) ** xx, np.where((xx + yy) % 4 < 2, 1.0, -1.0), np.where((xx - yy) % 4 < 2, 1.0, -1.0),
                     np.where(yy % 4 < 2, 1.0, -1.0), np.where(xx % 4 < 2, 1.0, -1.0)])
    wt = rng.random((n, 6)) ** rng.choice([1.0, 4.0, 12.0], size=(n, 1)) * (rng.random((n, 6)) < 0.7)
    amp = (pmax / 2) * 2.0 ** -rng.uniform(0, bd + 1, size=(n, 1, 1))
    cells = pmax / 2 + amp * np.tensordot(wt, pats, 1) + rng.integers(-1, 2, size=(n, 12, 12)) * rng.integers(0, 3, size=(n, 1, 1))
    steps = []
    for cv in alf_clip_values(bd):
        for d in (cv - 1, cv, cv + 1):
            d = min(d, pmax)
            for orient in range(2):
                s = np.where((xx if orient else yy) % 6 < 3, 0, d)
                steps += [s, pmax - s]
    return np.clip(np.rint(np.concatenate([cells, np.array(steps, float)])), 0, pmax).astype(np.int16)


def _mosaic(cells, rows, cols):
    m = np.zeros((rows * 12, cols * 12), np.int16)
    for i in range(rows * cols):
        r, c = divmod(i, cols)
        m[12 * r:12 * r + 12, 12 * c:12 * c + 12] = cells[i % len(cells)]
    return m


_alf_select_cache = {}


def _alf_select_cells(bd, seed=7, n=24000):
    """Pool cells whose centre 4x4 block (classified on the cell alone) adds a coverage key not seen before, in pool order."""
    if bd in _alf_select_cache: return _alf_select_cache[bd]
    pool = _alf_cell_pool(bd, n, seed)
    cols = 100
    rows = (len(pool) + cols - 1) // cols
    cs = alf_class_sums(_mosaic(pool, rows, cols), bd, 1 << 20)
    i = np.arange(len(pool))
    r, c = 3 * (i // cols) + 1, 3 * (i % cols) + 1
    cls, tr, act, cmp, nz = cs["cls"][r, c], cs["tr"][r, c], cs["act"][r, c], cs["cmp"][:, r, c], cs["nz"][:, r, c]
    seen, pick = set(), []
    for k in range(len(pool)):
        keys = {("ct", int(cls[k]), int(tr[k])), ("act", int(act[k]))} | {("cmp", j, int(cmp[j, k])) for j in range(5) if cmp[j, k] or nz[j, k]}
        if keys - seen: seen |= keys; pick.append(k)
    _alf_select_cache[bd] = (pool, pool[pick])
    return _alf_select_cache[bd]


def _alf_luma_content(kind, bd, ctu, W, H, rng):
    pmax = (1 << bd) - 1
    rows, cols = (H + 11) // 12, (W + 11) // 12
    pool, chosen = _alf_select_cells(bd)
    cells = [pool[int(i)] for i in rng.integers(0, len(pool), size=rows * cols)]
    if kind == "classes":                                   # the chosen cells where no virtual boundary row touches their windows
        slots = [(r, c) for r in range(rows) for c in range(cols) if 12 * r + 12 <= H and 12 * c + 12 <= W
                 and all(not (ctu - 12 <= y % ctu < ctu + 4) and y % ctu >= 4 for y in range(12 * r, 12 * r + 12))]
        assert len(slots) >= len(chosen), (len(slots), len(chosen))
        for k, (r, c) in enumerate(slots[:len(chosen)]): cells[r * cols + c] = chosen[k]
    elif kind in ("coeffs", "cc"):                          # 0 / pmax checkerboards (output and correction clips) between the texture cells
        yy, xx = np.mgrid[0:12, 0:12]
        board = np.where((xx + yy) % 2, pmax, 0).astype(np.int16)
        for i in range(0, len(cells), 3 if kind == "cc" else 5): cells[i] = board if (i // 5) % 2 else pmax - board
    return _mosaic(cells, rows, cols)[:H, :W]


def _alf_tables(bd, part, rng):
    """24 luma sets: the 16 fixed ones, then APS sets with +128 on every tap, one +128 per class (on tap class % 12), -128 / 127, all zero, the
    full int8 range, the range with +128, small, and a mix; clip indices rotating over taps and classes.  8 chroma alternatives with +-128 taps.
    4 CC-ALF filters per component whose 56 taps take the next 56 values of 0, 1, -1, ..., 64, -64 (part 0, 1, 2)."""
    clipv = alf_clip_values(bd)
    coef = np.zeros((24, 4, 25, 13), np.int16); clip = np.zeros((24, 4, 25, 13), np.int16)
    coef[:16] = _fixed_sets(); clip[:16] = clipv[0]
    k, t = np.arange(25)[:, None], np.arange(13)[None, :]
    one = rng.integers(-20, 21, size=(25, 13)); one[np.arange(25), np.arange(25) % 12] = 128
    mix = rng.integers(-128, 128, size=(25, 13)); mix[20:, 11] = 128
    bases = [np.full((25, 13), 128), one, np.where((k + t) % 2, 127, -128), np.zeros((25, 13), int), rng.integers(-128, 128, size=(25, 13)),
             rng.integers(-128, 129, size=(25, 13)), rng.integers(-8, 9, size=(25, 13)), mix]
    for s, base in enumerate(bases, 16):
        base = np.array(base); base[:, 12] = 128
        bclip = np.array(clipv)[(k + t + s) % 4]
        for tr in range(4):
            coef[s, tr] = base[:, ALF_TR[tr]]; clip[s, tr] = bclip[:, ALF_TR[tr]]
    a = np.arange(8)[:, None]; tt = np.arange(7)[None, :]
    cco = np.concatenate([np.full((1, 7), 128), np.full((1, 7), -128), np.where(tt % 2, 128, -128), np.zeros((1, 7), int),
                          rng.integers(-128, 129, size=(4, 7))]).astype(np.int16)
    cco[:, 6] = 128
    ccl = np.array(clipv)[(a + tt) % 4].astype(np.int16)
    vals = [0] + [v for m in range(1, 65) for v in (m, -m)]
    vals = (vals + [64, -64] * 30)[56 * part:56 * part + 56]
    cc = [np.array(vals[28 * c:28 * c + 28], np.int16).reshape(4, 7) for c in range(2)]
    return dict(lumaCoeff=np.ascontiguousarray(coef), lumaClip=np.ascontiguousarray(clip), chromaCoeff=cco, chromaClip=ccl, cc=cc)


def _alf_records(kind, ctusW, ctusH, sets):
    n = ctusW * ctusH
    i = np.arange(n)
    a = np.zeros(n, ALFCTU_DTYPE)
    a["enable"][:, 0] = i % 5 != 4                         # unfiltered CTUs next to filtered ones
    a["enable"][:, 1] = i % 3 != 2; a["enable"][:, 2] = i % 4 != 1
    a["lumaSet"] = np.array(sets)[i % len(sets)]
    a["chromaAlt"][:, 0] = i % 8; a["chromaAlt"][:, 1] = (i + 3) % 8
    a["ccIdx"][:, 0] = i % 5; a["ccIdx"][:, 1] = (i + 2) % 5
    if kind == "flags":                                     # every CLIP combination, corner padding and the wide chroma form where legal
        a["enable"][:, 0] = 1 | ((i % 16) << 1)
        cx, cy, f = i % ctusW, i // ctusW, (i % 16) << 1
        tl = (i % 3 == 0) & (f & (ALF_CLIP_TOP_ | ALF_CLIP_LEFT_) == 0) & (cx > 0) & (cy > 0)
        br = (i % 3 == 1) & (f & (ALF_CLIP_BOTTOM_ | ALF_CLIP_RIGHT_) == 0) & (cx < ctusW - 1) & (cy < ctusH - 1)
        a["enable"][:, 0] |= (tl * 32 + br * 64).astype(np.uint8)
        for c in range(2):
            wide = (a["ccIdx"][:, c] == 0) & (i % 2 == c)
            a["enable"][:, 1 + c] |= (wide * 2).astype(np.uint8)
    return a


ALF_CLIP_TOP_, ALF_CLIP_BOTTOM_, ALF_CLIP_LEFT_, ALF_CLIP_RIGHT_ = 2, 4, 8, 16

# name: (kind, bit depth, CTU, W, H, chroma, strides, CC-ALF coefficient part)
ALF_SWEEP_CASES = {
    "classes_8bit_ctu64": ("classes", 8, 64, 384, 256, True, None, 0),
    "classes_9bit_ctu128_last120": ("classes", 9, 128, 392, 376, True, None, 1),
    "classes_10bit_ctu128": ("classes", 10, 128, 384, 384, True, None, 2),
    "coeffs_10bit_ctu32_last24": ("coeffs", 10, 32, 264, 248, True, None, 0),
    "coeffs_8bit_ctu32": ("coeffs", 8, 32, 256, 256, True, None, 1),
    "ccalf_8bit_ctu128": ("cc", 8, 128, 264, 256, True, None, 0),
    "ccalf_9bit_ctu64": ("cc", 9, 64, 264, 192, True, None, 1),
    "ccalf_10bit_ctu32": ("cc", 10, 32, 264, 160, True, None, 2),
    "flags_10bit_ctu64": ("flags", 10, 64, 520, 320, True, None, 0),
    "flags_8bit_ctu32": ("flags", 8, 32, 264, 248, True, None, 1),
    "geometry_400_ctu64": ("classes", 10, 64, 256, 128, False, None, 0),
    "geometry_strides_ctu32": ("coeffs", 10, 32, 200, 136, True, (216, 108, 112), 2),
    "uhd_3840x2160": ("mix", 10, 128, 3840, 2160, True, None, 0),
}


def _alf_case(name):
    kind, bd, ctu, W, H, chroma, strides, part = ALF_SWEEP_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    pmax = (1 << bd) - 1
    luma = _alf_luma_content(kind, bd, ctu, W, H, rng)

    def content(c, w, h):
        if c == 0: return luma
        if kind == "cc":                                    # chroma at 0 / pmax / mid, so the corrected sample clips both ways
            return np.array([0, pmax, pmax // 2], np.int16)[rng.integers(0, 3, size=(h // 2 + 1, w // 2 + 1))].repeat(2, 0).repeat(2, 1)[:h, :w]
        pool = _alf_cell_pool(bd, 400, 100 + c)
        return _mosaic([pool[int(i)] for i in rng.integers(0, len(pool), size=((h + 11) // 12) * ((w + 11) // 12))], (h + 11) // 12, (w + 11) // 12)[:h, :w]
    planes = _k45_planes(W, H, chroma, strides, content)
    t = _alf_tables(bd, part, rng)
    ctusW, ctusH = (W + ctu - 1) // ctu, (H + ctu - 1) // ctu
    sets = list(range(24)) if kind in ("classes", "mix") else list(range(16, 24)) + [0, 15]
    t["ctus"] = _alf_records(kind, ctusW, ctusH, sets)
    if kind == "classes" and ctusW * ctusH < 24:            # every set on some CTU: fewer CTUs than sets in the small pictures, so rotate per case
        t["ctus"]["lumaSet"] = (np.arange(ctusW * ctusH) * 5 + part * 7) % 24
    g = abi.make_geom(W, H, bd, chroma_format=1 if chroma else 0, ctu=ctu, strides=strides)
    return dict(name=name, kind=kind, g=g, W=W, H=H, bd=bd, ctu=ctu, chroma=chroma, strides=strides, planes=planes, tables=t,
                flagged=bool((t["ctus"]["enable"][:, 0] & 0xfe).any() or (t["ctus"]["enable"][:, 1:] & 2).any()))


def _sao_content(kind, bd, w, h, rng):
    pmax = (1 << bd) - 1
    if kind == "bo":                                        # every band's first, second, middle and last value, and 0 / pmax
        bw = 1 << (bd - 5)
        vals = np.unique([0, pmax] + [v for k in range(32) for v in (k * bw, k * bw + 1, k * bw + bw // 2, (k + 1) * bw - 1)])
        return vals[rng.integers(0, len(vals), size=(h, w))]
    # three levels around a base that changes every 4x4 unit (low, high, middle): plateaus (sign 0), local extremes next to 0 and pmax
    base = np.array([0, pmax - 2, pmax // 2])[rng.integers(0, 3, size=(h // 4 + 1, w // 4 + 1))].repeat(4, 0).repeat(4, 1)[:h, :w]
    return base + rng.integers(0, 3, size=(h, w))


def _sao_records(kind, ctusW, ctusH, bd, chroma):
    n = ctusW * ctusH
    M = sao_max_offset(bd)
    s = np.zeros(n, SAO_DTYPE)
    s["type"] = 255
    s["avail"] = picture_avail(ctusW, ctusH)
    eo = [[M, M, 0, -M, -M], [1, M, 0, -M, -1], [M, 1, 0, -1, -M]]
    for i in range(n):
        for c in range(3 if chroma else 1):
            if kind == "bo" or (kind == "mix" and (i + c) % 4 == 0):
                sg = 1 if (i + c) % 2 else -1
                s["type"][i, c] = 4; s["band"][i, c] = (i + 11 * c) % 32; s["offset"][i, c, :4] = [sg * M, -sg * M, sg * M, -sg * M]
            elif kind == "mix" and (i + c) % 5 == 1:
                continue
            else:
                s["type"][i, c] = ((i // 256 if kind == "masks" else i) + c) % 4; s["offset"][i, c] = eo[(i + c) % 3]
    if kind == "masks":                                     # interior CTUs: every avail mask with every luma class
        cx, cy = np.arange(n) % ctusW, np.arange(n) // ctusW
        inner = np.flatnonzero((cx > 0) & (cx < ctusW - 1) & (cy > 0) & (cy < ctusH - 1))
        for k, i in enumerate(inner):
            s["avail"][i] = k % 256; s["type"][i, 0] = (k // 256) % 4
    return s


# name: (kind, bit depth, CTU, W, H, chroma, strides, (vertical VBs, horizontal VBs))
SAO_SWEEP_CASES = {
    "bo_8bit_ctu32": ("bo", 8, 32, 256, 128, True, None, ((), ())),
    "bo_9bit_ctu32": ("bo", 9, 32, 256, 128, True, None, ((), ())),
    "bo_10bit_ctu64": ("bo", 10, 64, 512, 256, True, None, ((), ())),
    "bo_12bit_ctu128": ("bo", 12, 128, 1024, 512, True, None, ((), ())),
    "eo_8bit_ctu32_partial": ("eo", 8, 32, 200, 136, True, None, ((), ())),
    "eo_10bit_ctu64_strides": ("eo", 10, 64, 424, 240, True, (440, 216, 220), ((), ())),
    "eo_12bit_ctu128": ("eo", 12, 128, 392, 264, True, None, ((), ())),
    "avail_masks_ctu32": ("masks", 10, 32, 1080, 1088, True, None, ((), ())),
    "vb_3x3_edges": ("eo", 10, 64, 384, 256, True, None, ((8, 128, 376), (8, 64, 248))),
    "vb_3x2_mod16": ("eo", 10, 32, 320, 192, True, None, ((24, 152, 296), (40, 88))),
    "vb_1x0_8bit": ("eo", 8, 128, 256, 128, True, None, ((136,), ())),
    "vb_0x2_12bit": ("eo", 12, 64, 256, 192, True, None, ((), (64, 184))),
    "vb_2x1_mix": ("mix", 10, 128, 512, 256, True, None, ((128, 264), (120,))),
    "geometry_400": ("mix", 10, 64, 256, 128, False, None, ((), ())),
    "geometry_400_stride": ("mix", 8, 32, 256, 128, False, (268, 0, 0), ((), ())),
    "uhd_3840x2160": ("mix", 10, 128, 3840, 2160, True, None, ((), ())),
}


def _sao_case(name):
    kind, bd, ctu, W, H, chroma, strides, (vx, vy) = SAO_SWEEP_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    planes = _k45_planes(W, H, chroma, strides, lambda c, w, h: _sao_content("bo" if kind == "bo" else "eo", bd, w, h, rng))
    ctusW, ctusH = (W + ctu - 1) // ctu, (H + ctu - 1) // ctu
    vb = abi.Vb()
    vb.numVer, vb.numHor = len(vx), len(vy)
    for k, x in enumerate(vx): vb.posX[k] = x
    for k, y in enumerate(vy): vb.posY[k] = y
    g = abi.make_geom(W, H, bd, chroma_format=1 if chroma else 0, ctu=ctu, strides=strides)
    return dict(name=name, kind=kind, g=g, W=W, H=H, bd=bd, ctu=ctu, chroma=chroma, strides=strides, planes=planes,
                ctus=_sao_records(kind, ctusW, ctusH, bd, chroma), vb=vb)


_k45_cache = {}


def sao_sweep(name):
    """One case of the designed K4 sweep (SAO_SWEEP_CASES): geometry (g, W, H, bd, ctu, chroma, strides), planes (stride padding holds -7), the CTU
    records and the virtual boundaries (abi.Vb).  bo: every band start 0..31 with samples on every band's edges, the largest legal offsets, 0 / pmax;
    eo: the four classes with plateaus and local extremes next to 0 / pmax, partial CTUs; masks: every avail mask with every luma class on interior
    CTUs; vb: 0..3 vertical and horizontal boundaries at 8, W - 8, on CTU edges and at 8 mod 16."""
    key = ("sao", name)
    if key not in _k45_cache: _k45_cache[key] = _sao_case(name)
    c = _k45_cache[key]
    return dict(c, planes=[p.copy() for p in c["planes"]], ctus=c["ctus"].copy())


def alf_sweep(name):
    """One case of the designed K5 sweep (ALF_SWEEP_CASES): geometry, planes (stride padding holds -7) and tables (synth.gen_alf's layout, ctus
    included).  classes: cells chosen to reach every class x transpose, activity and comparison side; coeffs: the scalar-path and int8-extreme APS
    sets on 0 / pmax checkerboards and clip steps; cc: every CC-ALF coefficient value over 0 / pmax luma and chroma; flags: every CLIP combination,
    PAD_TL / PAD_BR and PAD_WIDE.  flagged: whether any CTU has clip / pad flags."""
    key = ("alf", name)
    if key not in _k45_cache: _k45_cache[key] = _alf_case(name)
    c = _k45_cache[key]
    t = c["tables"]
    return dict(c, planes=[p.copy() for p in c["planes"]], tables=dict(t, ctus=t["ctus"].copy(), cc=[x.copy() for x in t["cc"]]))


# ---- what the library refuses: its kernel-level entry points check every rule (vvdec_b200/csrc/rules.cuh) on the host, before any device work, so
# these ask it on any machine.  Without a GPU a legal call returns B200_ERR_NO_DEVICE; on one it runs, on zero planes of the geometry.
def library_refusal(fn, *args):
    """The error message of the library's entry point `fn` when it refuses the call with `args` (B200_ERR_PARAM), else None."""
    from . import lib
    return lib().b200_last_error().decode() if getattr(lib(), fn)(*args) == -2 else None


def _zero_planes(g):
    return [np.zeros((g.height >> (c > 0), g.stride[c]), np.int16) if c == 0 or g.chromaFormat else None for c in range(3)]


def lf_problems(case):
    """What b200_lf_deblock says about a call of lf_sweep's form (g, lfV, lfH; ctuSlice, slices, seq and dirs default to none, one slice, no LADF and 3):
    [] when it accepts the call, else [its error message]."""
    k = dict(dict(ctuSlice=None, slices=np.zeros(1, LFSLICE_DTYPE), seq=abi.LfSeq(), dirs=3), **case)
    lfV, lfH, cs, planes = np.ascontiguousarray(k["lfV"]), np.ascontiguousarray(k["lfH"]), k["ctuSlice"], _zero_planes(k["g"])   # alive until the call returns
    msg = library_refusal("b200_lf_deblock", C.byref(k["g"]), abi.plane_ptrs(planes), lfV.ctypes.data, lfH.ctypes.data,
                          None if cs is None else cs.ctypes.data, k["slices"].ctypes.data, len(k["slices"]), C.addressof(k["seq"]), k["dirs"])
    return [] if msg is None else [msg]


def lf_grid_problems(grid, d, g):
    """What b200_lf_deblock says about the grid of direction d (0 lfV, 1 lfH) of geometry g, the other direction without edges."""
    z = np.zeros_like(grid)
    return lf_problems(dict(g=g, lfV=z if d else grid, lfH=grid if d else z))


def lf_grid_legal(grid, d, g):
    return not lf_grid_problems(grid, d, g)


def k45_record_problems(kind, g, ctus, tables=None, vb=None):
    """What b200_sao_picture (kind 'sao') / b200_alf_picture ('alf') says about a geometry, its CTU records and tables (gen_alf's layout: only the
    numbers of sets count) or virtual boundaries: [] when it accepts the call, else [its error message]."""
    src, dst = _zero_planes(g), _zero_planes(g)
    ctus = np.ascontiguousarray(ctus)
    if kind == "sao":
        msg = library_refusal("b200_sao_picture", C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(dst), ctus.ctypes.data, None if vb is None else C.addressof(vb))
    else:
        n = [tables["lumaCoeff"].shape[0], tables["chromaCoeff"].shape[0], tables["cc"][0].shape[0], tables["cc"][1].shape[0]]
        t = dict(lumaCoeff=np.zeros((n[0], 1300), np.int16), chromaCoeff=np.zeros((n[1], 7), np.int16), cc=[np.zeros((m, 7), np.int16) for m in n[2:]])
        t["lumaClip"], t["chromaClip"] = t["lumaCoeff"], t["chromaCoeff"]
        T = abi.make_alf_tables(t)
        msg = library_refusal("b200_alf_picture", C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(dst), ctus.ctypes.data, C.byref(T))
    return [] if msg is None else [msg]


def k1_record_problems(g, tus, coefs, scaling=None):
    """What b200_k1_residual says about a geometry, its TU records, level arena and scaling arena: [] when it accepts the call, else [its error message]."""
    planes, tus, coefs = _zero_planes(g), np.ascontiguousarray(tus), np.ascontiguousarray(coefs, np.int16)
    sl = None if scaling is None else np.ascontiguousarray(scaling, np.int32)
    msg = library_refusal("b200_k1_residual", C.byref(g), abi.plane_ptrs(planes), tus.ctypes.data, len(tus), coefs.ctypes.data, len(coefs),
                          None if sl is None else sl.ctypes.data, 0 if sl is None else len(sl), 0)
    return [] if msg is None else [msg]


# ---- K1: the designed residual sweep (tests/test_k1_*.py).  Each TU names what it is there for (tags) and, where the decoder can produce it, the
# syntax it comes from (tests.helpers.RefTuSyntax fields; tests/test_k1_oracle_vs_ref.py flattens it with the glue and runs it through the reference).
K1_TR_NAMES = {abi.TR_DCT2: "DCT2", abi.TR_DST7: "DST7", abi.TR_DCT8: "DCT8"}
K1_ODD = (1, 3, 5, 15, 31)
K1_SCAN = ((0, 0), (0, 1), (1, 0), (0, 2), (1, 1), (2, 0), (0, 3), (1, 2), (2, 1), (3, 0), (1, 3), (2, 2), (3, 1), (2, 3), (3, 2), (3, 3))   # (y, x) of the 16 LFNST inputs
# LFNST (set, transpose) -> an intra mode that selects it on a square block (H.266 lfnstTrSetIdx; modes above 34 transpose)
K1_LFNST_MODES = {(0, 0): 0, (1, 0): 8, (1, 1): 60, (2, 0): 18, (2, 1): 50, (3, 0): 34, (3, 1): 40}
# (zeroOutSize, outputs) -> the shapes with that LFNST form; the second list holds the dual-tree chroma shapes
K1_LFNST_SHAPES = {(8, 16): ([(4, 4)], [(4, 4)]), (8, 48): ([(8, 8)], [(8, 8)]),
                   (16, 16): ([(4, 8), (8, 4), (4, 16), (16, 4), (4, 32), (32, 4), (4, 64), (64, 4)], [(4, 8), (16, 4)]),
                   (16, 48): ([(16, 16), (8, 16), (16, 8), (32, 32), (64, 64), (8, 64), (64, 16)], [(16, 16), (32, 32), (8, 32)])}


def k1_tr_sides(n):
    """The 1-D transforms a side of n samples can take: DST-7 and DCT-8 exist for 4..32."""
    return (abi.TR_DCT2, abi.TR_DST7, abi.TR_DCT8) if 4 <= n <= 32 else (abi.TR_DCT2,)


def k1_zero_out(tr, n):
    """How many coefficients of a side can be coded: 16 for DST-7 / DCT-8 at 32, else min(n, 32)."""
    return 16 if tr != abi.TR_DCT2 and n == 32 else min(n, 32)


def k1_lfnst_form(w, h):
    """(zeroOutSize, outputs) of LFNST on a w x h block: 8 inputs on 4x4 and 8x8, 48 outputs when both sides are at least 8."""
    return (8 if (w, h) in ((4, 4), (8, 8)) else 16), (48 if w >= 8 and h >= 8 else 16)


class _K1Case:
    """TU records packed row by row into their planes (luma; one shelf for both chroma planes, so a joint-CbCr partner never overlaps another TU)."""
    def __init__(self, W, bd, rng):
        self.W, self.bd, self.rng = W, bd, rng
        self.recs, self.levels, self.tags, self.syntax, self.n = [], [], [], [], 0
        self.shelf = [[0, 0, 0], [0, 0, 0]]

    def place(self, comp, w, h):
        s, pw = self.shelf[comp > 0], self.W >> (comp > 0)
        if s[0] + w > pw: s[0], s[1], s[2] = 0, s[1] + s[2], 0
        x, y = s[0], s[1]
        s[0] += w; s[2] = max(s[2], h)
        return x, y

    def height(self):
        return max(8, self.shelf[0][1] + self.shelf[0][2], 2 * (self.shelf[1][1] + self.shelf[1][2]) + 8) + 7 & ~7

    def add(self, tag, comp, w, h, lv, qp, dq=False, tr=0, lfnst=0, ict=0, flags=0, sl_off=0, syntax=None, at=None, dqp=None):
        """qp = QP (QP' - 6 (bd - 8)); lv = the level corner (rows maxY + 1, columns maxX + 1).  A chroma TU with a syntax form keeps qp <= 26, where the
        default chroma QP mapping is the identity."""
        lv = np.asarray(lv, np.int16).reshape(np.shape(lv)[0], -1)
        l2w, l2h = w.bit_length() - 1, h.bit_length() - 1
        x, y = at or self.place(comp, w, h)
        rs, ib, sc = dqp or tu_dequant(qp + 6 * (self.bd - 8), self.bd, l2w, l2h, bool(flags & abi.TU_TS), dq, bool(flags & abi.TU_SCALING))
        self.recs.append((x, y, l2w, l2h, comp, flags, lv.shape[1] - 1, lv.shape[0] - 1, tr, lfnst, ict, rs, ib, sc, self.n, sl_off, (0, 0)))
        self.levels.append(lv.reshape(-1)); self.n += lv.size; self.tags.append(tag)
        self.syntax.append(None if syntax is None else dict(syntax, comp=comp, bitDepth=self.bd, qp=qp, depQuant=int(dq),
                                                            w=w << (comp > 0), h=h << (comp > 0)))

    def extreme(self, k, rows, cols):
        """Saturating levels whose signs follow a basis row: all +32767 / all -32768 (row 0 of DCT-2, DST-7 and DCT-8 has one sign), signs alternating
        by coefficient row or column (the last DCT-2 row), or a random sign per level."""
        yy, xx = np.mgrid[0:rows, 0:cols]
        sign = [np.ones_like(yy), -np.ones_like(yy), 1 - 2 * (yy & 1), 1 - 2 * (xx & 1), self.rng.choice([-1, 1], size=(rows, cols))][k % 5]
        return np.where(sign > 0, 32767, -32768)


def _k1_pair_syntax(w, h, trH, trV):
    """A luma syntax form that selects (trH, trV) on a w x h TU: DCT-2 on an inter CU, explicit MTS, or implicit MTS (DST-7 on sides 4..16 of an intra
    CU of at most 32x32, DCT-2 on the others); None where only SBT / ISP give the pair."""
    D2, S7, C8 = abi.TR_DCT2, abi.TR_DST7, abi.TR_DCT8
    if trH == D2 and trV == D2: return dict(predMode=0)
    if trH != D2 and trV != D2: return dict(predMode=1, spsMTS=1, spsIntraMTS=1, mtsIdx=2 + (trH == C8) + 2 * (trV == C8))
    if max(w, h) <= 32 and (trH == S7) == (w <= 16) and (trV == S7) == (h <= 16) and C8 not in (trH, trV):
        return dict(predMode=1, spsMTS=1, spsIntraMTS=0)
    return None


def _k1_pairs(b):
    """Every shape x every legal (trH, trV): DC only, the whole zero-out corner (random and saturating levels) and an odd corner."""
    k = 0
    for l2w in range(1, 7):
        for l2h in range(1, 7):
            w, h = 1 << l2w, 1 << l2h
            comp = 0 if min(w, h) >= 4 else 1 + (k & 1)                 # sides of 2 only exist in chroma
            for trH in k1_tr_sides(w):
                for trV in k1_tr_sides(h):
                    tr, zx, zy = trH | (trV << 2), k1_zero_out(trH, w), k1_zero_out(trV, h)
                    ox, oy = [v for v in K1_ODD if v <= zx], [v for v in K1_ODD if v <= zy]
                    ox, oy = ox[k % len(ox)], oy[(k // len(ox)) % len(oy)]
                    syn = _k1_pair_syntax(w, h, trH, trV) if comp == 0 else None
                    tag = f"pairs {w}x{h} {K1_TR_NAMES[trH]}x{K1_TR_NAMES[trV]}"
                    b.add(tag + " DC only", comp, w, h, [[int(b.rng.integers(1, 3000)) * (1 - 2 * (k & 1))]], 30, tr=tr, syntax=syn)
                    b.add(tag + " full", comp, w, h, b.rng.integers(-300, 301, (zy, zx)), 27, dq=bool(k & 1), tr=tr, syntax=syn)
                    b.add(tag + " full saturating", comp, w, h, b.extreme(k, zy, zx), 37, tr=tr, syntax=syn)
                    b.add(tag + f" odd corner {ox}x{oy}", comp, w, h, b.rng.integers(-300, 301, (oy, ox)), 32, tr=tr, syntax=syn)
                    k += 1


def _k1_lfnst(b):
    """Every (set, index, transpose) x every LFNST form x one-hot input at each of the 16 scan positions (corner 4x4 or just reaching the input), and all
    16 inputs saturated."""
    i = 0
    for form, (luma, chroma) in K1_LFNST_SHAPES.items():
        shapes = [(0, s) for s in luma] + [(1, s) for s in chroma]
        for (st, tp), mode in K1_LFNST_MODES.items():
            for idx in (1, 2):
                code = idx | (st << 2) | (tp << 4)
                for pos in range(17):
                    comp, (w, h) = shapes[i % len(shapes)]
                    comp = comp and 1 + (i & 1)
                    i += 1
                    if pos < 16:
                        y, x = K1_SCAN[pos]
                        lv = np.zeros((4, 4) if i & 1 else (y + 1, x + 1), np.int16)
                        lv[y, x] = int(b.rng.integers(50, 600)) * (1 - 2 * (pos & 1))
                        tag = f"lfnst set {st} idx {idx} transpose {tp} {w}x{h} input {pos}"
                    else:
                        lv, tag = b.extreme(i, 4, 4), f"lfnst set {st} idx {idx} transpose {tp} {w}x{h} all 16 inputs saturated"
                    pinned = w == h and (pos < form[0] or pos == 16)          # the parser never codes inputs past zeroOutSize
                    syn = dict(predMode=1, spsLFNST=1, lfnstIdx=idx, sepTree=int(comp > 0), intraDirL=mode, intraDirC=mode) if pinned else None
                    b.add(tag, comp, w, h, lv, 22 if pos < 16 else 26, lfnst=code, syntax=syn)


def _k1_dequant(b):
    """Every QP of the bit depth, with and without dependent quantisation, on 4x4 / 8x4 luma (all 12 scales) and 2x4 / 2x2 chroma (the most negative
    shifts): levels at +-inMax, +-(inMax + 1) and +-32768 through transform skip (the residual is the dequantised level), DC-only DCT-2 and full corners;
    every third QP also with a scaling list of entries 1 and 255; 2x2 records with shifts of -10..-12 and every scale, where the inMax clip binds."""
    bd = b.bd
    for qp in range(-6 * (bd - 8), 64):
        for dq in (False, True):
            for comp, w, h, kind in ((0, 4, 4, "ts"), (0, 4, 4, "dc"), (0, 8, 4, "dc"), (0, 4, 4, "full"), (1, 2, 4, "full"), (2, 2, 2, "full")):
                ts = kind == "ts"
                if ts and dq: continue
                rs, ib, _ = tu_dequant(qp + 6 * (bd - 8), bd, w.bit_length() - 1, h.bit_length() - 1, ts, dq)
                m = (1 << (ib - 1)) - 1
                vals = np.array([m, -m, min(m + 1, 32767), -m - 1, 32767, -32768, 1, -1], np.int64)
                lv = np.array([[vals[(qp + dq) % len(vals)]]]) if kind == "dc" else b.rng.choice(vals, size=(h, w))
                syn = dict(predMode=0, mtsIdx=int(ts)) if comp == 0 or (h == 4 and qp <= 26) else None
                tag = f"dequant QP {qp}{' depquant' if dq else ''} {w}x{h} {kind} rightShift {rs}"
                b.add(tag, comp, w, h, lv, qp, dq=dq, flags=abi.TU_TS if ts else 0, syntax=syn)
                if qp % 3 == 0 and comp == 0 and not ts:
                    b.add(tag + " scaling list 1 / 255", comp, w, h, lv, qp, dq=dq, flags=abi.TU_SCALING, sl_off=b.sl_off[(w, h)])
    # the inMax clip keeps level * scale << -rightShift inside 32 bits: shifts past the decoder's, with every scale (records only)
    for rs in (-10, -11, -12):
        for sc in sorted({s for row in TU_INV_SCALES for s in row}):
            lv = b.rng.choice([32767, -32768, 1 << (24 + rs), -(1 << (24 + rs)) - 1], size=(2, 2))
            b.add(f"dequant rightShift {rs} scale {sc}", 2, 2, 2, lv, 0, dqp=(rs, min(16, 25 + rs), sc))


def _k1_ts_bdpcm(b):
    """Transform skip at every size up to 32 (2xN / Nx2 chroma included), and BDPCM H and V whose lines of +32767 / -32768 saturate the running sum."""
    shapes = [(0, w, h) for w in (4, 8, 16, 32) for h in (4, 8, 16, 32)] + [(1, w, h) for w in (2, 4, 8, 16) for h in (2, 4, 8, 16)]
    for k, (comp, w, h) in enumerate(shapes):
        comp = comp and 1 + (k & 1)
        qp = 4 - 6 * (b.bd - 8)                                         # QP' 4: the dequantised level is the level
        syn = dict(predMode=0, mtsIdx=1)
        b.add(f"ts {w}x{h}", comp, w, h, b.rng.integers(-32768, 32768, (h, w)), qp, flags=abi.TU_TS, syntax=syn)
        b.add(f"ts {w}x{h} QP 25", comp, w, h, b.rng.integers(-400, 401, (h, w)), 25, flags=abi.TU_TS, syntax=syn)
        for mode, flag in ((1, abi.TU_BDPCM_H), (2, abi.TU_BDPCM_V)):
            n, length = (h, w) if mode == 1 else (w, h)
            lines = [np.full(length, 32767), np.full(length, -32768), np.where(np.arange(length) & 1, -32768, 32767),
                     np.where(np.arange(length) < length // 2, 32767, -32768), b.rng.integers(-20000, 20001, length)]
            lv = np.array([lines[(i + k) % len(lines)] for i in range(n)])
            lv = lv if mode == 1 else lv.T
            syn = dict(predMode=1, mtsIdx=1, **({"bdpcmL": mode} if comp == 0 else {"bdpcmC": mode}))
            for q in (qp, 25):
                b.add(f"bdpcm {'HV'[mode - 1]} {w}x{h} QP {q}", comp, w, h, lv, q, flags=abi.TU_TS | flag, syntax=syn)


def _k1_jccr(b):
    """Joint CbCr: every ict on Cb and on Cr, with residuals -32768, -1, +1, odd negatives and +32767 (transform skip at QP' 4) and transform blocks of
    saturating and random levels; run on predictions of 0 and pmax."""
    vals = np.array([-32768, -1, 1, -3, -5, -32767, 32767, 3, -7, 0], np.int64)
    k = 0
    for comp in (1, 2):
        for ict in (1, -1, 2, -2, 3, -3):
            for w, h in ((2, 2), (2, 4), (4, 2), (4, 4), (8, 8), (16, 16), (32, 32), (8, 2)):
                syn = dict(jointCbCr={1: 2, 2: 3, 3: 1}[abs(ict)], jointCbCrSign=int(ict < 0)) if (abs(ict) == 3) == (comp == 2) and (w, h) != (2, 2) else None
                tag = f"jccr ict {ict} comp {comp} {w}x{h}"
                b.add(tag + " ts", comp, w, h, b.rng.choice(vals, size=(h, w)), 4 - 6 * (b.bd - 8), ict=ict, flags=abi.TU_TS,
                      syntax=syn and dict(syn, predMode=0, mtsIdx=1))
                zx, zy = min(w, 32), min(h, 32)
                b.add(tag + " saturating", comp, w, h, b.extreme(k, zy, zx), 26, ict=ict, syntax=syn and dict(syn, predMode=0))
                b.add(tag + " random", comp, w, h, b.rng.integers(-900, 901, (zy, zx)), 24, ict=ict, dq=True, syntax=syn and dict(syn, predMode=0))
                k += 1


# name -> (kind, bit depth, width, height (None: as packed), 4:2:0?, strides or None, prediction)
K1_SWEEP_CASES = {
    "pairs_10bit": ("pairs", 10, 1024, None, True, (1029, 515, 517), "noise"),
    "lfnst_10bit": ("lfnst", 10, 1024, None, True, (1032, 516, 516), "noise"),
    "dequant_8bit": ("dequant", 8, 256, None, True, (260, 131, 130), "noise"),
    "dequant_9bit": ("dequant", 9, 256, None, True, None, "noise"),
    "dequant_10bit": ("dequant", 10, 256, None, True, (257, 128, 129), "noise"),
    "dequant_12bit": ("dequant", 12, 256, None, True, None, "extreme"),
    "ts_bdpcm_10bit": ("ts_bdpcm", 10, 512, None, True, (515, 257, 259), "noise"),
    "ts_bdpcm_8bit": ("ts_bdpcm", 8, 512, None, True, None, "extreme"),
    "jccr_10bit": ("jccr", 10, 512, None, True, (516, 259, 258), "extreme"),
    "jccr_12bit": ("jccr", 12, 512, None, True, None, "extreme"),
    "geometry_400": ("random", 10, 256, 136, False, (261, 0, 0), "noise"),
    "geometry_9bit_odd_strides": ("random", 9, 200, 136, True, (203, 101, 107), "noise"),
    "geometry_12bit_edges": ("random", 12, 392, 264, True, None, "extreme"),
    "uhd_3840x2160": ("random", 10, 3840, 2160, True, None, "noise"),
}


def _k1_case(name):
    import zlib
    kind, bd, W, H, chroma, strides, pred = K1_SWEEP_CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    scaling = None
    if kind == "random":
        # dense TUs of every kind over a whole partitioned picture: its last row and column included
        cus = partition(rng, W, H, ctu=128)
        tus, coefs = gen_tus(rng, cus, bd, p_cbf=0.9, p_mts=0.25, p_lfnst=0.2, p_ts=0.15, p_bdpcm=0.1, p_jccr=0.3, p_full=0.8, chroma=chroma,
                             heavy=0.3, p_intra=0.6)
        tags, syntax = ["geometry"] * len(tus), [None] * len(tus)
    else:
        b = _K1Case(W, bd, rng)
        if kind == "dequant":
            b.sl_off = {(4, 4): 0, (8, 4): 16}
            scaling = np.where((np.arange(48) + np.arange(48) // 4) & 1, 255, 1).astype(np.int32)
        {"pairs": _k1_pairs, "lfnst": _k1_lfnst, "dequant": _k1_dequant, "ts_bdpcm": _k1_ts_bdpcm, "jccr": _k1_jccr}[kind](b)
        H = b.height()
        tus, coefs, tags, syntax = np.array(b.recs, abi.TU_DTYPE), np.concatenate(b.levels), b.tags, b.syntax
    pmax = (1 << bd) - 1

    def content(c, w, h):
        if pred == "noise": return noise_planes(rng, w, h, bd, chroma=False)[0]
        yy, xx = np.mgrid[0:h, 0:w]                                     # 4x4 blocks of 0 and pmax, Cr the inverse of Cb
        return np.where(((yy >> 2) + (xx >> 2) + (c == 2)) & 1, pmax, 0)
    planes = _k45_planes(W, H, chroma, strides, content)
    if not chroma: planes += [None, None]
    g = abi.make_geom(W, H, bd, chroma_format=1 if chroma else 0, strides=strides)
    return dict(name=name, kind=kind, g=g, W=W, H=H, bd=bd, chroma=chroma, strides=strides, planes=planes, tus=tus, coefs=coefs, scaling=scaling,
                tags=tags, syntax=syntax)


_k1_cache = {}


def k1_sweep(name):
    """One case of the designed K1 sweep (K1_SWEEP_CASES): geometry (g, W, H, bd, chroma, strides), prediction planes (stride padding holds -7; None for
    absent chroma), TU records, level arena, scaling arena (or None), per-TU tags and syntax (None: a record only the record interface allows).
    pairs: every shape x (trH, trV) with DC-only, zero-out and odd corners and saturating levels; lfnst: every set / index / transpose x LFNST form x
    input position; dequant: every QP, both quantisers, all scales, the most negative shifts, inMax and scaling-list extremes; ts_bdpcm: transform skip
    at every size and saturating BDPCM lines; jccr: every ict on both chroma planes over 0 / pmax predictions; geometry: 4:0:0, odd strides, picture
    edges, 4K."""
    if name not in _k1_cache: _k1_cache[name] = _k1_case(name)
    c = _k1_cache[name]
    return dict(c, planes=[None if p is None else p.copy() for p in c["planes"]])


def k1_corner(tus, coefs, i):
    """The level corner of TU i: (maxY + 1, maxX + 1) int16."""
    t = tus[i]
    mx, my, off = int(t["maxX"]) + 1, int(t["maxY"]) + 1, int(t["coefOff"])
    return coefs[off:off + mx * my].reshape(my, mx)


def k1_lmcs_picture(ctu, W=256, H=128, bd=10):
    """TUs and prediction for LMCS chroma residual scaling on the picture path: luma constant per VPDU, at values spread over the LMCS bins, so that the
    VPDUs' neighbourhoods pick different chromaAdjHelpLUT entries; in each VPDU's chroma area a 2x2 TU (never scaled), 2x4 and 4x2 TUs, 4x4 / 8x8 TUs and
    joint-CbCr pairs (transform skip with the level as residual, and DCT-2), and one luma TU.  Returns (tus, coefs, given planes, tags)."""
    import zlib
    rng = np.random.default_rng(zlib.crc32(f"lmcs{ctu}".encode()))
    b = _K1Case(W, bd, rng)
    vs = 64 if ctu == 128 else ctu
    pmax = (1 << bd) - 1
    luma = np.zeros((H, W), np.int16)
    ts = dict(flags=abi.TU_TS, qp=4 - 6 * (bd - 8))
    for k, (vy, vx) in enumerate((vy, vx) for vy in range(0, H, vs) for vx in range(0, W, vs)):
        luma[vy:vy + vs, vx:vx + vs] = 24 + ((k * 7) % 16) * ((pmax - 48) // 15)
        cx, cy, ict = vx // 2, vy // 2, (1, -1, 2, -2, 3, -3)[k % 6]
        for comp, w, h, dx, dy, kw in ((1, 2, 2, 0, 0, ts), (2, 2, 4, 2, 0, ts), (1, 4, 2, 4, 0, ts), (1 + (abs(ict) == 3), 4, 4, 8, 0, dict(ts, ict=ict)),
                                        (2, 4, 4, 12, 0, dict(qp=27)), (1 + (abs(ict) == 3), 8, 8, 0, 8, dict(qp=24, ict=-ict)), (1, 8, 8, 8, 8, ts)):
            lv = rng.integers(-300, 301, (h, w))
            b.add(f"lmcs VPDU {k} comp {comp} {w}x{h}{' ict %d' % kw['ict'] if 'ict' in kw else ''}", comp, w, h, lv, at=(cx + dx, cy + dy), **kw)
        b.add(f"lmcs VPDU {k} luma 8x8", 0, 8, 8, rng.integers(-40, 41, (8, 8)), 30, at=(vx + 8, vy + 8))
    chroma = [(pmax // 2 + rng.integers(-100, 101, (H // 2, W // 2))).astype(np.int16) for _ in range(2)]
    return np.array(b.recs, abi.TU_DTYPE), np.concatenate(b.levels), [luma] + chroma, b.tags
