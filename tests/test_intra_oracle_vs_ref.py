"""K6 intra prediction (SURVEY 8f-1, regular modes): the oracle against the real IntraPrediction (reference sample derivation, [1 2 1] filter,
planar / DC / angular incl. wide angles / MRL / PDPC / BDPCM prediction; C and SIMD kernels), on random CU layouts where the predicted CU has
whatever neighbourhood the decoding order gives it.  The records come from the glue flattener (flatten_intra.h), whose availability counts the
shim checks against IntraPrediction::m_neighborSize."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth

pytestmark = pytest.mark.ref

CHROMA_MODES = [0, 1, 18, 50, 2, 34, 66, 70, 70, 70, 23, 45, 61]       # 70 = DM (PU::getFinalIntraMode -> the luma mode)


def run_case(oracle, ref, rng, W, H, bd, ctu, simd, layout, k, dirL, dirC, mrl, bdpcm, bdpcmC=0, mip=0, colloc=0, paint=None, out=None, resi=None):
    """paint(planes): writes designed neighbour samples into the noise planes before the reference runs; out: a list the reference's planes are
    appended to; resi: residual planes the predicted CU adds (clip(pred + resi)), else prediction only."""
    g = abi.make_geom(W, H, bd, ctu=ctu)
    planes = synth.noise_planes(rng, W, H, bd)
    if paint: paint(planes)
    cus = np.zeros(k + 1, synth.REF_INTRA_CU_DTYPE)
    for i in range(k + 1):
        cus[i]["x"], cus[i]["y"], cus[i]["w"], cus[i]["h"] = layout[i]
        cus[i]["dirL"], cus[i]["dirC"] = 0, 0
    cus[k]["dirL"], cus[k]["dirC"], cus[k]["multiRefIdx"], cus[k]["bdpcm"], cus[k]["bdpcmC"] = dirL, dirC, mrl, bdpcm, bdpcmC
    x, y, w, h = layout[k]
    luma_only = w < 8 or (w // 2) * (h // 2) < 16                       # such luma blocks are CUs of a local dual tree: no chroma of their own
    cus[k]["rsv"][0] = luma_only
    cus[k]["rsv"][2] = mip                                           # bit 0 MIP (dirL = MIP mode index), bit 1 transposed
    cus[k]["rsv"][1] = resi is not None                              # add the residual
    want = [p.copy() for p in planes]
    recs = np.zeros(3, abi.INTRA_TU_DTYPE)
    n = ref.ref_intra_case(simd, C.byref(g), abi.plane_ptrs(want), None if resi is None else abi.plane_ptrs(resi), cus.ctypes.data, k + 1, 0, recs.ctypes.data, 3, colloc)
    assert n == (1 if luma_only else 3), n
    recs = recs[:n]
    got = [p.copy() for p in planes]
    if resi is None: oracle.orc_intra_predict(C.byref(g), abi.plane_ptrs(got), recs.ctypes.data, n)
    else: oracle.orc_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), recs.ctypes.data, n)
    for c in range(3):
        assert np.array_equal(got[c], want[c]), (c, layout[k], dirL, dirC, mrl, bdpcm, recs[c])
    assert not np.array_equal(want[0][y:y + h, x:x + w], planes[0][y:y + h, x:x + w])
    # the synthetic generator used by the GPU tests derives the same records (availability from the decoding order, filter decision, DM)
    mine = synth.gen_intra_records(rng, layout, W, H, modes={k: (dirL, dirC, mrl, bdpcm, mip)}, upto=k, colloc=colloc)
    mine = mine[-n:]
    if resi is not None: mine["flags"] |= abi.INTRA_ADD_RESI
    for f in ("x", "y", "log2w", "log2h", "comp", "mode", "multiRefIdx", "flags", "numAbove", "numLeft", "mip", "lmAbove", "lmLeft"):
        assert np.array_equal(mine[f], recs[f]), (f, mine[f], recs[f], layout[k])
    if out is not None: out.append(want)
    return recs


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("W,H,bd,ctu,seed", [(256, 128, 10, 128, 1), (192, 128, 10, 64, 2), (256, 128, 8, 128, 3), (136, 72, 10, 64, 4), (256, 256, 12, 128, 5)])
def test_intra_random_layouts(oracle, ref, W, H, bd, ctu, seed, simd):
    if simd and bd > 10: pytest.skip("the x86 chroma kernels multiply in 16 bit: exact up to 10 bit (Main10), the C kernels are the 12-bit reference")
    rng = np.random.default_rng(seed)
    seen = set()
    for it in range(60):
        layout = synth.gen_intra_layout(rng, W, H, ctu, min_size=8 if it % 3 else 4, p_split=0.6 + 0.3 * rng.random())
        k = 0 if it == 0 else int(rng.integers(len(layout)))           # it 0: the first CU of the picture has no neighbours at all
        if it == 1: k = next(i for i, c in enumerate(layout) if c[1] == 0 and c[0] > 0)      # top picture edge: left only
        if it == 2: k = next(i for i, c in enumerate(layout) if c[0] == 0 and c[1] > 0)      # left picture edge: above only
        x, y, w, h = layout[k]
        kind = it % 6
        dirL, mrl, bdpcm = int(rng.integers(0, 67)), 0, 0
        if kind == 4: mrl, dirL = int(rng.integers(1, 3)), int(rng.integers(1, 67))
        if kind == 5 and w <= 32 and h <= 32: bdpcm = int(rng.integers(1, 3))
        if kind == 0: dirL = int(rng.integers(0, 2))
        dirC = CHROMA_MODES[int(rng.integers(len(CHROMA_MODES)))]
        recs = run_case(oracle, ref, rng, W, H, bd, ctu, simd, layout, k, dirL, dirC, mrl, bdpcm)
        seen.add((int(recs[0]["numAbove"]) > 0, int(recs[0]["numLeft"]) > 0, bool(recs[0]["flags"] & 2)))
    assert len(seen) >= 4                                              # corner / edge / interior neighbourhoods all occurred


@pytest.mark.parametrize("w,h", [(4, 4), (4, 16), (16, 4), (8, 32), (32, 8), (64, 64), (64, 16), (16, 64), (8, 8), (4, 32), (32, 4), (64, 8), (8, 64)])
def test_intra_all_modes_per_shape(oracle, ref, w, h):
    """Every mode (incl. the wide-angle remapped ones) and both MRL lines for each block shape, interior position, C kernels and SIMD kernels."""
    rng = np.random.default_rng(w * 131 + h)
    W, H, ctu = 256, 128, 128
    # hand-made layout: the block at (64, 64) with everything before it in decoding order present
    layout = [(0, 0, 64, 64), (64, 0, 64, 64), (0, 64, 64, 64), (64, 64, w, h)]
    for mode in range(67):
        for mrl in (0, 1, 2):
            if mrl and (mode == 0 or (mode + mrl) % 4): continue          # planar has no MRL; sample the rest
            if (w == 4 or h == 4) and False: continue
            run_case(oracle, ref, rng, W, H, 10, ctu, (mode + mrl) & 1, layout, 3, mode, CHROMA_MODES[mode % len(CHROMA_MODES)], mrl, 0)


from tests.helpers import intra_picture_case


@pytest.mark.parametrize("W,H,bd,ctu,simd,seed", [(256, 128, 10, 128, 1, 11), (192, 128, 10, 64, 0, 12), (416, 240, 8, 128, 1, 13), (256, 256, 12, 128, 0, 14)])
def test_intra_picture_chain(oracle, ref, W, H, bd, ctu, simd, seed):
    rng = np.random.default_rng(seed)
    g, planes, resi, recs, want = intra_picture_case(ref, rng, W, H, bd, ctu, simd, colloc=seed & 1, min_size=8)
    assert (recs["mode"] >= abi.INTRA_LM).any() and (recs["mode"] == abi.INTRA_MIP).any()
    got = [p.copy() for p in planes]
    oracle.orc_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), recs.ctypes.data, len(recs))
    for c in range(3):
        assert np.array_equal(got[c], want[c]), c
    assert (recs["flags"] & 4).any() and not (recs["flags"] & 4).all()


@pytest.mark.parametrize("w,h", [(4, 4), (4, 8), (8, 4), (8, 8), (4, 16), (16, 4), (16, 16), (8, 16), (32, 8), (32, 32), (64, 64), (64, 16), (16, 64), (8, 32), (64, 32)])
def test_intra_mip_all_modes(oracle, ref, w, h):
    """Matrix intra prediction: every mode of the block's size class, plain and transposed, interior and picture-corner positions."""
    rng = np.random.default_rng(w * 7 + h)
    W, H, ctu = 256, 128, 128
    n_modes = 16 if (w, h) == (4, 4) else 8 if (w == 4 or h == 4 or (w, h) == (8, 8)) else 6
    for layout, k in (([(0, 0, 64, 64), (64, 0, 64, 64), (0, 64, 64, 64), (64, 64, w, h)], 3), ([(0, 0, w, h)], 0), ([(0, 0, 64, 64), (64, 0, w, h)], 1)):
        for mode in range(n_modes):
            for tr in (0, 1):
                run_case(oracle, ref, rng, W, H, 10 if mode % 2 else 8, ctu, mode & 1, layout, k, mode, 70, 0, 0, mip=1 | (tr << 1))


@pytest.mark.parametrize("colloc", [0, 1])
@pytest.mark.parametrize("w,h", [(8, 8), (16, 16), (32, 32), (64, 64), (16, 8), (8, 16), (64, 16), (16, 64), (32, 8), (8, 32), (16, 4), (64, 32)])
def test_intra_cclm(oracle, ref, w, h, colloc):
    """Cross-component linear model (LM, MDLM_L, MDLM_T): luma down-sampling (3 / 5 / 6 tap: first CTU row, collocated chroma, default), template
    selection and parameter derivation, for interior blocks, CTU-row starts and picture edges (no left / no above neighbour)."""
    rng = np.random.default_rng(w * 5 + h + colloc)
    W, H, ctu = 256, 256, 128
    layouts = [([(0, 0, 64, 64), (64, 0, 64, 64), (0, 64, 64, 64), (64, 64, w, h)], 3),          # interior
               ([(0, 0, 128, 64), (0, 64, 64, 64), (64, 64, 64, 64), (0, 128, w, h)], 3) if False else ([(0, 0, 64, 64), (64, 0, 64, 64), (0, 64, 64, 64), (64, 64, 64, 64), (0, 128, w, h)], 4),   # first row of a CTU, left picture edge
               ([(0, 0, w, h)], 0),                                                               # picture corner: no template at all
               ([(0, 0, 64, 64), (64, 0, w, h)], 1)]                                              # top picture edge: left only
    for layout, k in layouts:
        for mode in (67, 68, 69):
            for rep in range(3):
                run_case(oracle, ref, rng, W, H, 10 if rep else 8, ctu, rep & 1, layout, k, int(rng.integers(0, 67)), mode, 0, 0, colloc=colloc)


@pytest.mark.parametrize("colloc", [0, 1])
@pytest.mark.parametrize("bd,simd", [(8, 0), (8, 1), (10, 0), (10, 1), (12, 0)])
def test_intra_cclm_designed(oracle, ref, bd, simd, colloc):
    """CCLM on designed neighbour planes (synth.cclm_target_values painted as the GPU sweep paints them): every target of the parameter derivation
    (every weak ordering of the four selected luma samples with distinct chroma, diff == 0, diffC == 0, each normDiff with either sign of diffC, the
    slope clamped to +-15) with LM (two above + two left), MDLM_T (four above) and MDLM_L (four left), and the three orderings of the two-sample path;
    the co-located luma is the reference's planar prediction over the designed rows and columns.  The 12-bit case runs the C kernels only (see
    test_intra_random_layouts)."""
    from tests.helpers import cclm_params
    rng = np.random.default_rng(bd * 4 + simd * 2 + colloc)
    W, H, ctu = 256, 256, 128
    interior = ([(0, 0, 64, 64), (64, 0, 64, 64), (0, 64, 64, 64), (64, 64, 16, 16)], 3)
    two = ([(0, 0, 64, 64), (64, 0, 16, 4)], 1)                      # top picture edge: 8x2 chroma with a left template of two samples
    jobs = [(interior, dirC, t) for dirC in (67, 68, 69) for t in synth.CCLM_TARGETS if t[0] in ("tie", "diff0", "diffC0", "normDiff", "clamp")]
    jobs += [(two, 67, ("tie2", o)) for o in range(3)]
    reached = set()
    for (layout, k), dirC, t in jobs:
        mine = synth.gen_intra_records(rng, layout, W, H, modes={k: (0, dirC, 0, 0, 0)}, upto=k, colloc=colloc)[-2]
        x, y, w, h = int(mine["x"]), int(mine["y"]), 1 << int(mine["log2w"]), 1 << int(mine["log2h"])
        sel_l, sel_c = synth.cclm_target_values(t, bd)
        want = []
        recs = run_case(oracle, ref, rng, W, H, bd, ctu, simd, layout, k, 0, dirC, 0, 0, colloc=colloc, out=want,
                        paint=lambda planes: synth.cclm_paint(planes, x, y, w, h, mine, sel_l, sel_c, bd))
        p = cclm_params(oracle, abi.make_geom(W, H, bd, ctu=ctu), want[0], recs[1])
        sl = list(p.selL)
        got = {"tie": ("tie",) + tuple(sorted(set(sl)).index(v) for v in sl), "tie2": ("tie2", 0 if sl[1] < sl[0] else 1 if sl[1] == sl[0] else 2),
               "diff0": ("diff0",) if p.maxL == p.minL else None, "diffC0": ("diffC0",) if p.maxC == p.minC and p.maxL > p.minL else None,
               "normDiff": ("normDiff", p.normDiff, 1 if p.maxC > p.minC else -1), "clamp": ("clamp", 1 if p.a > 0 else -1) if p.clamped else None}[t[0]]
        assert got == t, (dirC, t, got, sl)
        reached.add((dirC, t))
    assert len(reached) == len(jobs)


def _designed_jobs(bd):
    """(w, h, dirL, mrl, bdpcm, mip, pattern, value, where, residual) of the designed regular-intra blocks run through the reference: the blocks of
    synth.intra_designed_sweep's targets and flat cases, at the position the layout gives them.  Every target x shape class is kept: cubic modes with
    MRL 0 / 1 / 2 and PDPC of modes 18 / 50 on every luma shape (chroma: the same modes as DM), BDPCM H / V, every MIP mode of one shape per size class
    (plain and transposed, both patterns; 4x64 and 64x4 up-sample by 16), no neighbour at the picture corner and padding from the left column at the top edge; flat references on
    every shape with a sample of modes.  Residuals of +-3/4 pmax on the pdpc, BDPCM and substitution blocks."""
    out = []
    pmax, mid = (1 << bd) - 1, 1 << (bd - 1)
    for i, (w, h) in enumerate(synth.INTRA_LUMA_SHAPES):
        for mrl in (0, 1, 2):
            if mrl and h == 64: continue                             # the interior position is not on the first row of a CTU, but keep the CTU case's rule
            out += [(w, h, m, mrl, 0, 0, "cubic", 0, "inner", False) for m in synth.intra_cubic_modes(w, h, mrl)[:2]]
        out += [(w, h, m, 0, 0, 0, "pdpc", 0, "inner", True) for m in (18, 50)]
        if w <= 32 and h <= 32: out += [(w, h, 0, 0, b, 0, "bdpcm", 0, "inner", True) for b in (1, 2)]
        out += [(w, h, (1, 66, 2)[i % 3], 0, 0, 0, None, 0, "corner", True), (w, h, (0, 50, 18)[i % 3], 0, 0, 0, "pad", (0, pmax)[i & 1], "top", True)]
        fm = [0, 1, 2, 18, 34, 50, 66] + [3 + (7 * i + 5 * j) % 63 for j in range(4)]
        out += [(w, h, m, (j % 3) * (m > 1 and h < 64), 0, 0, "flat", (0, 1, mid, pmax - 1, pmax)[(i + j) % 5], "inner", False) for j, m in enumerate(fm)]
    for (w, h) in ((4, 4), (8, 8), (16, 16), (4, 64), (64, 4)):       # 4x64 / 64x4: up-sampling by 16, which wraps the reference's int16 sums at 12 bit
        out += [(w, h, m, 0, 0, 1 | (tr << 1), p, 0, "inner", False) for m in range(synth.intra_mip_modes(w, h)) for tr in (0, 1) for p in ("mip_a", "mip_b")]
    return out


@pytest.mark.parametrize("bd,simd", [(8, 0), (8, 1), (10, 0), (10, 1), (12, 0)])
def test_intra_designed_vs_ref(oracle, ref, bd, simd):
    """Regular intra prediction on the designed references of synth.intra_designed_sweep (the targets and flat cases), painted around the predicted
    CU, the reference's planes against the oracle's (prediction, or pred + resi where a residual is given).  Every clip site reaches below 0 and above
    pmax, substitution takes the mid value and pads 0 / pmax, as the oracle's probe says.  The 12-bit case runs the C kernels only (see
    test_intra_random_layouts)."""
    from tests.helpers import intra_probes
    rng = np.random.default_rng(bd * 2 + simd)
    W, H, ctu = 256, 128, 128
    pmax = (1 << bd) - 1
    layouts = {"inner": ([(0, 0, 64, 64), (64, 0, 64, 64), (0, 64, 64, 64)], (64, 64)), "corner": ([], (0, 0)), "top": ([(0, 0, 64, 64)], (64, 0))}
    reached = set()
    for (w, h, dirL, mrl, bdpcm, mip, pattern, v, where, add) in _designed_jobs(bd):
        before, (x, y) = layouts[where]
        layout = before + [(x, y, w, h)]

        def paint(planes):
            if pattern is None: return
            pat = synth._intra_pattern(pattern, bd, v)
            synth._intra_paint(planes[0], x, y, w, h, 4, pat)
            for c in (1, 2): synth._intra_paint(planes[c], x // 2, y // 2, max(w // 2, 2), max(h // 2, 2), 2, pat)
        resi = [rng.integers(-(3 * pmax) // 4, (3 * pmax) // 4 + 1, size=(H >> (c > 0), W >> (c > 0))).astype(np.int16) for c in range(3)] if add else None
        want = []
        recs = run_case(oracle, ref, rng, W, H, bd, ctu, simd, layout, len(before), dirL, 70, mrl, bdpcm, mip=mip, paint=paint, out=want, resi=resi)
        before_planes = [p.copy() for p in want[0]]                  # the probe re-runs the records over the reference's output, where the neighbours are unchanged
        g = abi.make_geom(W, H, bd, ctu=ctu)
        for r, p in zip(recs, intra_probes(oracle, g, before_planes, recs, resi)):
            c = int(r["comp"]) > 0
            if p.cubicMin < 0: reached.add(("cubic_lo", mrl))
            if p.cubicMax > pmax: reached.add(("cubic_hi", mrl))
            if p.pdpcMin < 0: reached.add(("pdpc_lo", c))
            if p.pdpcMax > pmax: reached.add(("pdpc_hi", c))
            if p.mipSizeId >= 0 and p.mipMin < 0: reached.add(("mip_lo", p.mipSizeId))
            if p.mipSizeId >= 0 and p.mipMax > pmax: reached.add(("mip_hi", p.mipSizeId))
            if (p.substMin, p.substMax) == (1 << (bd - 1),) * 2 and r["numAbove"] + r["numLeft"] == 0: reached.add(("subst_mid", c))
            if pattern == "pad" and (p.substMin, p.substMax) == (v, v): reached.add(("pad", v, c))
            if resi is not None and p.recoMin < 0: reached.add(("reco_lo", c))
            if resi is not None and p.recoMax > pmax: reached.add(("reco_hi", c))
            if pattern == "flat": assert (p.predMin, p.predMax) == (v, v), (r, v)
    want = {(t, m) for t in ("cubic_lo", "cubic_hi") for m in (0, 1, 2)} | {(t, c) for t in ("pdpc_lo", "pdpc_hi", "subst_mid", "reco_lo", "reco_hi") for c in (False, True)}
    want |= {(t, s) for t in ("mip_lo", "mip_hi") for s in range(3)} | {("pad", v, c) for v in (0, pmax) for c in (False, True)}
    assert want <= reached, sorted(want - reached)


@pytest.mark.parametrize("w,h", [(8, 8), (16, 16), (32, 32), (64, 64), (16, 8), (8, 16), (64, 16), (16, 64), (32, 8), (4, 16), (16, 4)])
def test_ciip_blend(oracle, ref, w, h):
    """CIIP: the block holds an inter prediction; planar intra prediction (filtered references for luma blocks > 32 samples, PDPC) blended with weights
    that depend on whether the left / above neighbour CUs are intra.  All four neighbour combinations, C and SIMD kernels, 8 / 10 bit."""
    rng = np.random.default_rng(w * 9 + h)
    W, H, ctu = 256, 128, 128
    for inter_mask in range(4):                                        # bit 0: left neighbour CU is inter, bit 1: above neighbour CU is inter
        layout = [(0, 0, 64, 64), (64, 0, 64, 64), (0, 64, 64, 64), (64, 64, w, h)]
        g = abi.make_geom(W, H, 10 if inter_mask & 1 else 8, ctu=ctu)
        planes = synth.noise_planes(rng, W, H, g.bitDepth)
        cus = np.zeros(4, synth.REF_INTRA_CU_DTYPE)
        for i, c in enumerate(layout): cus[i]["x"], cus[i]["y"], cus[i]["w"], cus[i]["h"] = c
        cus[2]["rsv"][2] = 8 if inter_mask & 1 else 0                  # (0, 64): the left neighbour
        cus[1]["rsv"][2] = 8 if inter_mask & 2 else 0                  # (64, 0): the above neighbour
        cus[3]["rsv"][2] = 4
        chroma_ok = (w // 2) > 2
        want = [p.copy() for p in planes]
        recs = np.zeros(3, abi.INTRA_TU_DTYPE)
        n = ref.ref_intra_case(inter_mask & 1, C.byref(g), abi.plane_ptrs(want), None, cus.ctypes.data, 4, 0, recs.ctypes.data, 3, 0)
        assert n == (3 if chroma_ok else 1), n
        recs = recs[:n]
        assert (recs["ciip"] == 3 - (inter_mask & 1) - (inter_mask >> 1)).all() and (recs["mode"] == 0).all()
        got = [p.copy() for p in planes]
        oracle.orc_intra_predict(C.byref(g), abi.plane_ptrs(got), recs.ctypes.data, n)
        for c in range(3):
            assert np.array_equal(got[c], want[c]), (c, inter_mask)
        assert not np.array_equal(want[0][64:64 + h, 64:64 + w], planes[0][64:64 + h, 64:64 + w])


@pytest.mark.parametrize("w,h", [(4, 8), (8, 4), (8, 8), (4, 16), (16, 4), (8, 16), (16, 8), (16, 16), (32, 8), (8, 32), (32, 32), (64, 64), (64, 16), (16, 64), (4, 32), (32, 4)])
def test_intra_isp_luma(oracle, ref, w, h):
    """Intra sub-partitions (groundwork for the next K6 slice): the oracle's ISP restatement against the real initIntraPatternChTypeISP / predIntraAng
    walk of DecCu — both split directions, partitions 1 / 2 samples thin (4-wide prediction regions), residual added on some partitions, interior /
    edge / corner CUs, planar, DC and angular modes (wide angles by the CU shape)."""
    rng = np.random.default_rng(w * 3 + h)
    W, H, ctu = 256, 128, 128
    layouts = [([(0, 0, 64, 64), (64, 0, 64, 64), (0, 64, 64, 64), (64, 64, w, h)], 3), ([(0, 0, w, h)], 0), ([(0, 0, 64, 64), (64, 0, w, h)], 1), ([(0, 0, 64, 64), (0, 64, w, h)], 1)]
    modes = [0, 1, 2, 18, 34, 50, 66] + [int(m) for m in rng.integers(2, 67, size=8)]
    for isp in (1, 2):
        split, non = (h, w) if isp == 1 else (w, h)
        part = max(split >> 2, 16 // non if non < 16 else 1)
        if part < 1 or split // part < 2: continue
        for layout, k in layouts:
            for mode in modes:
                bd = 10 if mode % 2 else 8
                g = abi.make_geom(W, H, bd, ctu=ctu)
                planes = synth.noise_planes(rng, W, H, bd)
                resi = [rng.integers(-30, 31, size=p.shape).astype(np.int16) for p in planes]
                cus = np.zeros(k + 1, synth.REF_INTRA_CU_DTYPE)
                for i in range(k + 1): cus[i]["x"], cus[i]["y"], cus[i]["w"], cus[i]["h"] = layout[i]
                mask = int(rng.integers(0, 16))
                cus[k]["dirL"], cus[k]["rsv"][2], cus[k]["bdpcmC"], cus[k]["rsv"][0] = mode, isp << 4, mask, 1      # luma-only CU (chroma goes the regular way)
                want = [p.copy() for p in planes]
                rec = np.zeros(1, abi.INTRA_TU_DTYPE)
                n = ref.ref_intra_case(mode & 1, C.byref(g), abi.plane_ptrs(want), abi.plane_ptrs(resi), cus.ctypes.data, k + 1, 0, rec.ctypes.data, 1, 0)
                assert n == 1, n
                r = rec[0]
                got = planes[0].copy()
                x, y = layout[k][0], layout[k][1]
                oracle.orc_intra_isp_cu(C.byref(g), got, resi[0].ctypes.data, x, y, w, h, isp, mode, int(bool(r["flags"] & 2)), int(r["numAbove"]), int(r["numLeft"]),
                                        int(r["lmLeft"]), int(r["lmAbove"]), mask)
                assert np.array_equal(got, want[0]), (isp, layout[k], mode, mask)
