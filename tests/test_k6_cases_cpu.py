"""The K6 test lists reach what tests/test_k6_intra_gpu.py claims they reach (no device needed): the designed sweep holds every block it lists and no
block of it reads another, and the generated cases put more than 1024 records into one CTU, stay below the density threshold where they stand for a B
picture, and never use MRL on the first row of a CTU.  The designed CCLM sweep reaches every geometry and parameter-derivation target it claims (as the
oracle derives them), and the rules refuse each malformed CCLM record on the host.  The designed sweep of regular modes (synth.intra_designed_sweep)
reaches every clip and substitution target it claims, as the oracle's own prediction reports them (orc_intra_probe)."""
import ctypes as C
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth
from tests import helpers


def test_designed_sweep_covers_its_list():
    W, H, recs = synth.intra_sweep()
    want = set(synth.intra_sweep_blocks())
    keys = [synth.intra_record_key(r) for r in recs]
    assert set(keys) == want
    # every block once per neighbourhood: full (the straight-copy fetch), partial (substitution), none
    full = {k for k, r in zip(keys, recs) if r["flags"] & abi.INTRA_AVAIL_TL}
    unit = np.where(recs["comp"] > 0, 2, 4)
    n_full = 2 * (1 << recs["log2w"].astype(int)) // unit + 2 * (1 << recs["log2h"].astype(int)) // unit
    total = recs["numAbove"].astype(int) + recs["numLeft"].astype(int)
    assert full == want and len(recs) == 3 * len(want)
    assert np.array_equal((recs["flags"] & abi.INTRA_AVAIL_TL) != 0, total == n_full)
    assert {k for k, t in zip(keys, total) if t == 0} == want
    partial = [(k, r) for k, r, t, n in zip(keys, recs, total, n_full) if 0 < t < n]
    assert {k for k, _ in partial} == want
    assert any(r["numAbove"] < 2 * (1 << int(r["log2w"])) // (2 if r["comp"] else 4) for _, r in partial)
    assert any(r["numLeft"] < 2 * (1 << int(r["log2h"])) // (2 if r["comp"] else 4) for _, r in partial)
    # shapes, modes and wide-angle remaps
    luma = {(w, h) for (c, w, h, *_) in want if c == 0}
    chroma = {(c, w, h) for (c, w, h, *_) in want if c}
    assert len(luma) == 25 and len(chroma) == 32
    for c, w, h in [(0, w, h) for (w, h) in luma] + sorted(chroma):
        assert all((c, w, h, m, 0, 0) in want for m in range(67))
        for m in range(2, 67):
            if synth.intra_wide_angle(w, h, m) != m: assert (c, w, h, m, 0, 0) in want
    remaps = {(w, h, m) for (c, w, h, m, mrl, mip) in want if m <= 66 and synth.intra_wide_angle(w, h, m) != m}
    assert len(remaps) > 100
    assert all((0, w, h, m, mrl, 0) in want for (w, h) in luma for mrl in (1, 2) for m in range(2, 67))
    assert all((0, w, h, abi.INTRA_MIP, 0, k | (t << 7)) in want for (w, h) in luma for t in (0, 1)
               for k in range(16 if (w, h) == (4, 4) else 8 if (w == 4 or h == 4 or (w, h) == (8, 8)) else 6))
    assert any(r["flags"] & abi.INTRA_FILTER_REF for r in recs)


def test_designed_sweep_is_independent_and_in_ctu_order():
    """No block's reference samples (row above incl. above-right and the corner, column left incl. below-left, MRL lines) are samples of another block:
    the sweep has no dependencies.  Records are in CTU raster order, every block inside its CTU."""
    W, H, recs = synth.intra_sweep()
    ctu = 128
    key = ((recs["y"].astype(np.int64) << (recs["comp"] > 0)) // ctu) * (W // ctu) + ((recs["x"].astype(np.int64) << (recs["comp"] > 0)) // ctu)
    assert np.all(np.diff(key) >= 0)
    for c in range(3):
        r = recs[recs["comp"] == c]
        pw, ph = (W, H) if c == 0 else (W // 2, H // 2)
        cs = ctu >> (1 if c else 0)
        occ = np.zeros((ph, pw), bool)
        for t in r:
            x, y, w, h = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"])
            assert x // cs == (x + w - 1) // cs and y // cs == (y + h - 1) // cs
            assert not occ[y:y + h, x:x + w].any()
            occ[y:y + h, x:x + w] = True
        for t in r:
            x, y, w, h, m = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"]), int(t["multiRefIdx"])
            assert x + 2 * w <= pw and y + 2 * h <= ph
            assert not occ[y - 1 - m:y, x - 1 - m:x + 2 * w].any() and not occ[y - 1 - m:y + 2 * h, x - 1 - m:x].any(), (c, x, y, w, h)


def test_generator_cases_reach_their_regime():
    counts = {}
    for name in ("ctu_1244_blocks", "ctu_1024_blocks", "sparse_1080p", "ctu64_200x136", "stride_420", "stride_417", "yuv400_8bit"):
        kw = helpers.INTRA_CASES[name]
        g, planes, resi, recs = helpers.intra_case(**kw)
        counts[name] = helpers.intra_ctu_counts(recs, kw["ctu"], kw["W"]).max()
        if name == "sparse_1080p":
            assert not helpers.intra_dense(g, len(recs))                          # v1 under auto
            assert set(np.unique(recs["ciip"][recs["ciip"] > 0]).tolist()) == {1, 2, 3}
        if name == "stride_420": assert all(s % 8 and not s % 2 for s in g.stride)
        if name == "stride_417": assert all(s % 2 for s in g.stride)
        if name == "yuv400_8bit": assert (recs["comp"] == 0).all() and planes[1] is None and g.chromaFormat == 0
        if name == "ctu64_200x136": assert ((recs["comp"] > 0) & (recs["x"] >= 96)).any() and ((recs["comp"] > 0) & (recs["y"] >= 64)).any()   # the 4-sample chroma tiles
    assert counts["ctu_1244_blocks"] > 1024                                          # records past the 1024 the CTU-resident kernel stages
    assert counts["ctu_1024_blocks"] == 1024


@pytest.mark.parametrize("ctu", [32, 64, 128])
def test_no_mrl_on_the_first_row_of_a_ctu(ctu):
    for seed in range(4):
        rng = np.random.default_rng(seed)
        layout = synth.gen_intra_layout(rng, 416, 240, ctu, min_size=4)
        recs = synth.gen_intra_records(rng, layout, 416, 240, p_mrl=0.5, ctu=ctu)
        mrl = recs[recs["multiRefIdx"] > 0]
        assert len(mrl) > 20 and not (mrl["y"] % ctu == 0).any()


# ---- the designed CCLM sweep (synth.cclm_sweep): what each case reaches, classified by the oracle's own derivation (orc_cclm_params)
def _cclm_reached(p, bd):
    """The targets (synth.CCLM_TARGETS, and ("tie2", order) on the two-sample path) one record reaches, and which selection it took."""
    pmax, sl, n = (1 << bd) - 1, list(p.selL), p.cntT + p.cntL
    out = set()
    if n == 4: out.add(("tie",) + tuple(sorted(set(sl)).index(v) for v in sl))
    if n == 2: out.add(("tie2", 0 if sl[1] < sl[0] else 1 if sl[1] == sl[0] else 2))   # the pair (s0, s1) comes back as s1, s0, s1, s0
    if n and p.maxL == p.minL: out.add(("diff0",))
    if p.maxL > p.minL and p.maxC == p.minC: out.add(("diffC0",))
    if p.normDiff >= 0 and p.maxC != p.minC: out.add(("normDiff", p.normDiff, 1 if p.maxC > p.minC else -1))
    if p.clamped and p.a: out.add(("clamp", 1 if p.a > 0 else -1))
    ends = [((p.a * v) >> p.shift) + p.b for v in (p.blkMin, p.blkMax)]
    if min(ends) < 0: out.add(("clip0",))
    if max(ends) > pmax: out.add(("clipmax",))
    if p.blkMin == 0: out.add(("luma0",))
    if p.blkMax == pmax: out.add(("lumamax",))
    sel = "2+2" if (p.cntT, p.cntL) == (2, 2) else "above" if p.cntT == 4 else "left" if p.cntL == 4 else "two" if n == 2 else "none"
    return sel, out


def _rules_accept(case):
    g, recs = case["g"], case["recs"]
    planes = [None if p is None else p.copy() for p in case["planes"]]
    rc = vvdec_b200.lib().b200_intra_reconstruct(C.byref(g), abi.plane_ptrs(planes), abi.plane_ptrs(case["resi"]), recs.ctypes.data, len(recs))
    assert rc in (0, -3), vvdec_b200.lib().b200_last_error()               # -3: no device (the host checks every record first)


@pytest.mark.parametrize("name", [n for n in synth.CCLM_SWEEP_CASES if n.startswith("targets")])
def test_cclm_targets_reached(oracle, name):
    """Every target of the parameter derivation is reached with two above + two left, four above and four left, and the two-sample path takes its
    three orderings; every block reaches what it was built for."""
    case = synth.cclm_sweep(name)
    g, bd = case["g"], case["bd"]
    seen = {}
    for r, tag in zip(case["recs"], case["tags"]):
        sel, got = _cclm_reached(helpers.cclm_params(oracle, g, case["planes"], r), bd)
        assert tag in got, (name, tag, sel, sorted(got), r)
        seen.setdefault(sel, set()).update(got)
    for sel in ("2+2", "above", "left"):
        assert set(synth.CCLM_TARGETS) <= seen[sel], (sel, sorted(set(synth.CCLM_TARGETS) - seen[sel]))
    assert {("tie2", o) for o in range(3)} <= seen["two"]
    assert len([t for t in synth.CCLM_TARGETS if t[0] == "tie"]) == 75
    _rules_accept(case)


@pytest.mark.parametrize("name", [n for n in synth.CCLM_SWEEP_CASES if n.startswith("geometry")])
def test_cclm_geometry_covered(name):
    """Every chroma shape that fits the chroma CTU, with every LM / MDLM neighbourhood, under the 3-tap (first row of a CTU), 5-tap (collocated) and
    6-tap filters; blocks without a left / above CU at the picture's left / top edge."""
    case = synth.cclm_sweep(name)
    recs, ctu, C = case["recs"], case["ctu"], case["ctu"] // 2
    have = set()
    for r in recs:
        w, h, fl = 1 << int(r["log2w"]), 1 << int(r["log2h"]), int(r["flags"])
        nb = (int(r["mode"]), int(bool(fl & abi.INTRA_LM_ABOVE)), int(bool(fl & abi.INTRA_LM_LEFT)), int(r["lmAbove"]), int(r["lmLeft"]), int(r["numAbove"]), int(r["numLeft"]))
        first = bool(fl & abi.INTRA_LM_ABOVE) and (2 * int(r["y"])) % ctu == 0
        have.add((w, h, nb, first, bool(fl & abi.INTRA_LM_COLLOCATED)))
        if r["x"] == 0: have.add((w, h, "left_edge"))
        if r["y"] == 0 and fl & abi.INTRA_LM_COLLOCATED: have.add((w, h, "top_edge"))
    shapes = [(w, h) for (w, h) in synth.CCLM_SHAPES if w <= C and h <= C]
    assert len(synth.CCLM_SHAPES) == 19 and (ctu < 64 or len(shapes) == 19)
    for (w, h) in shapes:
        nbs = synth.cclm_neighbourhoods(w, h)
        for nb in nbs:
            # the above template of a block as high as the chroma CTU always lies on the first row of a CTU (3-tap)
            for first, colloc in [(h == C and bool(nb[1]), 0), (h == C and bool(nb[1]), 1)] + ([(True, 0), (True, 1)] if nb[1] else []):
                if first and not colloc and (w, h, nb, True, True) in have and h < C: continue       # the first row is taken once, collocated or not
                assert (w, h, nb, first, bool(colloc)) in have or (first and (w, h, nb, True, not colloc) in have), (w, h, nb, first, colloc)
        assert (w, h, "left_edge") in have and (w, h, "top_edge") in have
        for mode, k in ((abi.INTRA_MDLM_T, 3), (abi.INTRA_MDLM_L, 4)):
            n, m = (w, h) if mode == abi.INTRA_MDLM_T else (h, w)
            lm = {nb[k] for nb in nbs if nb[0] == mode}
            assert {0, n // 2, n // 2 + min(n // 2, m // 2)} <= lm and len(lm) >= min(4, 2 + (min(n // 2, m // 2) >= 2))
    _rules_accept(case)


@pytest.mark.parametrize("name", [n for n in synth.CCLM_SWEEP_CASES if n != "chained"])
def test_cclm_sweep_is_independent_and_in_ctu_order(name):
    """No block's chroma reference samples (2w above incl. the corner, 2h left) are another block's samples, records are in CTU raster order, every
    block inside its chroma CTU; the list holds chroma records only, so the luma every block reads is the planes' own."""
    case = synth.cclm_sweep(name)
    recs, W, ctu = case["recs"], case["W"], case["ctu"]
    assert (recs["comp"] > 0).all() and (recs["mode"] >= abi.INTRA_LM).all()
    key = ((recs["y"].astype(np.int64) * 2) // ctu) * (W // ctu) + (recs["x"].astype(np.int64) * 2) // ctu
    assert np.all(np.diff(key) >= 0)
    cs = ctu // 2
    for c in (1, 2):
        r = recs[recs["comp"] == c]
        occ = np.zeros((case["H"] // 2, W // 2), bool)
        for t in r:
            x, y, w, h = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"])
            assert x // cs == (x + w - 1) // cs and y // cs == (y + h - 1) // cs
            assert not occ[y:y + h, x:x + w].any()
            occ[y:y + h, x:x + w] = True
        for t in r:
            x, y, w, h = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"])
            assert not occ[max(0, y - 1):y, max(0, x - 1):x + 2 * w].any() and not occ[max(0, y - 1):y + 2 * h, max(0, x - 1):x].any(), (c, x, y, w, h)


def test_cclm_chained_depends_on_earlier_luma(oracle):
    """The chained case: every CCLM block selects other template luma, and predicts something else in Cb or Cr, when the luma blocks before it are
    left out; its templates come from luma blocks in the CTU above and in the CTU to the left."""
    case = synth.cclm_sweep("chained")
    g, recs, planes, ctu = case["g"], case["recs"], case["planes"], case["ctu"]
    full = [p.copy() for p in planes]
    oracle.orc_intra_predict(C.byref(g), abi.plane_ptrs(full), recs.ctypes.data, len(recs))
    only = np.ascontiguousarray(recs[recs["comp"] > 0])
    alone = [p.copy() for p in planes]
    oracle.orc_intra_predict(C.byref(g), abi.plane_ptrs(alone), only.ctypes.data, len(only))
    luma = np.ascontiguousarray(recs[recs["comp"] == 0])
    lumad = [p.copy() for p in planes]
    oracle.orc_intra_predict(C.byref(g), abi.plane_ptrs(lumad), luma.ctypes.data, len(luma))
    assert len(only) >= 10
    for t in only:
        x, y, w, h = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"])
        assert list(helpers.cclm_params(oracle, g, lumad, t).selL) != list(helpers.cclm_params(oracle, g, planes, t).selL), (x, y)
        assert any(not np.array_equal(full[c][y:y + h, x:x + w], alone[c][y:y + h, x:x + w]) for c in (1, 2)), (x, y)
        cx, cy = 2 * x // ctu, 2 * y // ctu
        assert (((luma["x"] // ctu) == cx) & ((luma["y"] // ctu) == cy - 1)).any() and (((luma["x"] // ctu) == cx - 1) & ((luma["y"] // ctu) == cy)).any()
    assert list(np.flatnonzero(recs["comp"] > 0)) != list(range(len(only)))   # luma records come first within each CTU
    _rules_accept(case)


@pytest.mark.parametrize("row", range(len(helpers.cclm_refusal_rows()[2])))
def test_cclm_refusals_on_the_host(row):
    """Each malformed CCLM record is refused before any device work, with the planes unchanged; the valid list is accepted."""
    g, ok, rows = helpers.cclm_refusal_rows()
    name, bad, what = rows[row]
    lib = vvdec_b200.lib()
    planes = [np.full((256 >> (c > 0), 256 >> (c > 0)), 100 + c, np.int16) for c in range(3)]
    resi = [np.ones_like(p) for p in planes]
    lst = np.ascontiguousarray(np.concatenate([ok, bad.reshape(1)]))
    got = [p.copy() for p in planes]
    assert lib.b200_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), lst.ctypes.data, len(lst)) == -2, name
    assert what.encode() in lib.b200_last_error(), (name, lib.b200_last_error())
    assert all(np.array_equal(a, b) for a, b in zip(got, planes))
    assert lib.b200_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), ok.ctypes.data, len(ok)) in (0, -3)


# ---- the designed sweep of regular modes (synth.intra_designed_sweep): what each case reaches, as the oracle's prediction reports it (orc_intra_probe)
def _intra_reached(case, oracle):
    """{(target, class)} the records of a case reach: the clip sites below 0 / above pmax per shape class, substitution values, pred + resi per
    component, BDPCM predictions at 0 and pmax."""
    pmax, mid = (1 << case["bd"]) - 1, 1 << (case["bd"] - 1)
    got = set()
    for r, tag, p in zip(case["recs"], case["tags"], helpers.intra_probes(oracle, case["g"], case["planes"], case["recs"], case["resi"])):
        c, w, h, mrl = int(r["comp"]), 1 << int(r["log2w"]), 1 << int(r["log2h"]), int(r["multiRefIdx"])
        if p.interp == 1 and p.cubicMin < 0: got.add(("cubic_lo", (w, h, mrl)))
        if p.interp == 1 and p.cubicMax > pmax: got.add(("cubic_hi", (w, h, mrl)))
        if p.pdpcMin < 0: got.add(("pdpc_lo", (c > 0, w, h, int(r["mode"]))))
        if p.pdpcMax > pmax: got.add(("pdpc_hi", (c > 0, w, h, int(r["mode"]))))
        if p.mipSizeId >= 0 and p.mipMin < 0: got.add(("mip_lo", (p.mipSizeId, int(r["mip"]) >> 7)))
        if p.mipSizeId >= 0 and p.mipMax > pmax: got.add(("mip_hi", (p.mipSizeId, int(r["mip"]) >> 7)))
        if p.mipSizeId >= 0: assert p.mipInput0 == ((1 << (case["bd"] - 1)) - p.mipInputOffset if p.mipSizeId < 2 else 0)
        edge = "top" if r["y"] == 0 else "left" if r["x"] == 0 else "inner"
        if (p.substMin, p.substMax) == (mid, mid) and r["numAbove"] + r["numLeft"] == 0: got.add(("subst_mid", (c > 0, edge)))
        if (p.substMin, p.substMax) == (0, 0) and tag[0] == "pad": got.add(("pad_0", (c > 0, edge)))
        if (p.substMin, p.substMax) == (pmax, pmax) and tag[0] == "pad": got.add(("pad_max", (c > 0, edge)))
        if p.recoMin < 0: got.add(("reco_lo", c))
        if p.recoMax > pmax: got.add(("reco_hi", c))
        if r["mode"] in (abi.INTRA_BDPCM_HOR, abi.INTRA_BDPCM_VER) and (p.predMin, p.predMax) == (0, pmax): got.add(("bdpcm", (int(r["mode"]), w, h)))
    return got


@pytest.mark.parametrize("name", [n for n, v in synth.INTRA_SWEEP_CASES.items() if v[0] == "targets"])
def test_intra_targets_reached(oracle, name):
    """Every target of INTRA_TARGETS in every shape class the case holds: the cubic interpolation below 0 and above pmax for every luma shape with
    MRL 0 (where the shape has a fractional cubic mode), 1 and 2; PDPC of modes 18 and 50 below 0 and above pmax on every luma and chroma shape; the
    reduced MIP prediction below 0 and above pmax in every size class, transposed and not; the mid value without neighbours, and padding at 0 and pmax
    from one unit, inside the picture and at its top and left edges; pred + resi below 0 and above pmax in every component; BDPCM H / V at 0 and pmax."""
    case = synth.intra_designed_sweep(name)
    ctu, chroma = case["ctu"], case["planes"][1] is not None
    got = _intra_reached(case, oracle)
    luma = [(w, h) for (w, h) in synth.INTRA_LUMA_SHAPES if w <= ctu and h <= ctu]
    shapes = [(False, w, h) for (w, h) in luma] + ([(True, w, h) for (w, h) in synth.INTRA_CHROMA_SHAPES if w <= ctu // 2 and h <= ctu // 2] if chroma else [])
    want = {(t, (w, h, mrl)) for t in ("cubic_lo", "cubic_hi") for (w, h) in luma for mrl in (0, 1, 2)
            if synth.intra_cubic_modes(w, h, mrl) and not (mrl and h == ctu)}
    want |= {(t, (c, w, h, m)) for t in ("pdpc_lo", "pdpc_hi") for (c, w, h) in shapes for m in (18, 50)}
    want |= {(t, (s, tr)) for t in ("mip_lo", "mip_hi") for s in range(3) for tr in (0, 1)}
    want |= {(t, (c, e)) for t in ("subst_mid", "pad_0", "pad_max") for c in ({False, True} if chroma else {False}) for e in ("inner", "top", "left")}
    want -= {("pad_0", (c, "top")) for c in (False, True)} | {("pad_max", (c, "left")) for c in (False, True)}   # the edge blocks pad from pmax at the top, 0 at the left
    want |= {(t, c) for t in ("reco_lo", "reco_hi") for c in (range(3) if chroma else range(1))}
    want |= {("bdpcm", (m, w, h)) for m in (abi.INTRA_BDPCM_HOR, abi.INTRA_BDPCM_VER) for (w, h) in luma if w <= 32 and h <= 32}
    assert len([t for t in want if t[0] == "cubic_lo"]) >= len(luma) * 2
    assert want <= got, sorted(want - got)
    assert {t for t, _ in got} == set(synth.INTRA_TARGETS)
    if "stride" in name: assert all(s % 2 for s in case["g"].stride)
    if "yuv400" in name: assert case["g"].chromaFormat == 0 and (case["recs"]["comp"] == 0).all()
    _rules_accept(case)


@pytest.mark.parametrize("name", [n for n, v in synth.INTRA_SWEEP_CASES.items() if v[0] == "flat"])
def test_intra_flat_predicts_its_value(oracle, name):
    """Every block of a flat case predicts its value v in every sample, for each v in {0, 1, mid, pmax - 1, pmax}, with full and cut neighbourhoods,
    through planar, DC, every angular mode on every shape, MRL 1 and 2, BDPCM; the angular modes take both the cubic and the Gaussian filter, and the
    filtered reference."""
    case = synth.intra_designed_sweep(name)
    bd, recs = case["bd"], case["recs"]
    probes = helpers.intra_probes(oracle, case["g"], case["planes"], recs)
    seen, interp = set(), {}
    for r, v, p in zip(recs, case["flat"], probes):
        assert (p.predMin, p.predMax) == (v, v), (r, v, p.predMin, p.predMax)
        c, w, h, m = int(r["comp"]), 1 << int(r["log2w"]), 1 << int(r["log2h"]), int(r["mode"])
        seen.add((c, w, h, m, int(r["multiRefIdx"])))
        interp.setdefault(m, set()).add(p.interp + 4 * p.filtered)
    pmax = (1 << bd) - 1
    assert set(case["flat"]) == {0, 1, 1 << (bd - 1), pmax - 1, pmax}
    for c, shapes in ((0, synth.INTRA_LUMA_SHAPES), (1, synth.INTRA_CHROMA_SHAPES), (2, synth.INTRA_CHROMA_SHAPES)):
        for (w, h) in shapes:
            assert all((c, w, h, m, 0) in seen for m in range(67)), (c, w, h)
            if c == 0: assert {mrl for (cc, ww, hh, m, mrl) in seen if (cc, ww, hh) == (0, w, h)} == ({0, 1, 2} if h < case["ctu"] else {0})
            if c == 0 and w <= 32 and h <= 32: assert {(0, w, h, abi.INTRA_BDPCM_HOR, 0), (0, w, h, abi.INTRA_BDPCM_VER, 0)} <= seen
    assert sum(1 for m in range(2, 67) if {1, 2} <= interp[m]) > 50           # most angular modes take both filters (on different shapes)
    assert any(5 in interp[m] or 4 in interp[m] for m in range(2, 67))       # angular modes on the filtered reference
    assert {(int(r["numAbove"]) < 2 * (1 << int(r["log2w"])) // (2 if r["comp"] else 4)) for r in recs} == {False, True}
    _rules_accept(case)


@pytest.mark.parametrize("name", [n for n in synth.INTRA_SWEEP_CASES if n != "regular_chained"])
def test_intra_designed_cases_are_independent_and_in_ctu_order(name):
    """No block's reference footprint (4 luma / 2 chroma rows above from the corner to 2w, as many columns left down to 2h) holds another block's
    samples; records are in CTU raster order, every block inside its CTU, MRL never on the first row of a CTU."""
    case = synth.intra_designed_sweep(name)
    recs, W, H, ctu = case["recs"], case["W"], case["H"], case["ctu"]
    key = ((recs["y"].astype(np.int64) << (recs["comp"] > 0)) // ctu) * (W // ctu) + ((recs["x"].astype(np.int64) << (recs["comp"] > 0)) // ctu)
    assert np.all(np.diff(key) >= 0)
    assert not (recs["y"][recs["multiRefIdx"] > 0] % ctu == 0).any()
    for c in range(3 if case["planes"][1] is not None else 1):
        r = recs[recs["comp"] == c]
        gap, cs, pw, ph = (2, ctu // 2, W // 2, H // 2) if c else (4, ctu, W, H)
        occ = np.zeros((ph, pw), bool)
        for t in r:
            x, y, w, h = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"])
            assert x // cs == (x + w - 1) // cs and y // cs == (y + h - 1) // cs
            assert not occ[y:y + h, x:x + w].any()
            occ[y:y + h, x:x + w] = True
        for t in r:
            x, y, w, h = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"])
            assert x + 2 * w <= pw and y + 2 * h <= ph
            assert not occ[max(0, y - gap):y, max(0, x - gap):x + 2 * w].any() and not occ[max(0, y - gap):y + 2 * h, max(0, x - gap):x].any(), (c, x, y, w, h)


def test_intra_chained_depends_on_its_producers(oracle):
    """The chained case: leaving out any one producer changes its consumer's prediction (the last above-right unit, the last below-left unit, the
    corner, MRL line 2); producers sit in the CTU above, the CTU to the left, the CTU above-right, the CTU above-left and the consumer's own CTU."""
    case = synth.intra_designed_sweep("regular_chained")
    g, recs, planes, tags, ctu = case["g"], case["recs"], case["planes"], case["tags"], case["ctu"]
    full = [p.copy() for p in planes]
    oracle.orc_intra_predict(C.byref(g), abi.plane_ptrs(full), recs.ctypes.data, len(recs))
    where = set()
    for i, tag in enumerate(tags):
        if tag[0] != "producer": continue
        j = tags.index(("consumer",) + tag[1:])
        assert j > i
        cons, prod = recs[j], recs[i]
        less = np.ascontiguousarray(np.delete(recs, i))
        got = [p.copy() for p in planes]
        oracle.orc_intra_predict(C.byref(g), abi.plane_ptrs(got), less.ctypes.data, len(less))
        x, y, w, h = int(cons["x"]), int(cons["y"]), 1 << int(cons["log2w"]), 1 << int(cons["log2h"])
        assert not np.array_equal(got[0][y:y + h, x:x + w], full[0][y:y + h, x:x + w]), tag
        where.add((tag[1], (int(prod["x"]) // ctu - x // ctu, int(prod["y"]) // ctu - y // ctu)))
    owner = np.full(planes[0].shape, len(recs))                      # no block claims a neighbour that a later block writes (a decoding order)
    for i, t in enumerate(recs): owner[int(t["y"]):int(t["y"]) + (1 << int(t["log2h"])), int(t["x"]):int(t["x"]) + (1 << int(t["log2w"]))] = i
    for i, t in enumerate(recs):
        x, y, m, na, nl = int(t["x"]), int(t["y"]), int(t["multiRefIdx"]), 4 * int(t["numAbove"]), 4 * int(t["numLeft"])
        reads = np.concatenate([owner[y - 1 - m:y, x:x + na].ravel(), owner[y:y + nl, x - 1 - m:x].ravel(), owner[y - 1 - m:y, x - 1 - m:x].ravel()])
        assert not ((reads > i) & (reads < len(recs))).any(), i
    assert {d for _, d in where} == {(1, -1), (-1, 0), (-1, -1), (0, -1), (0, 0)}
    assert {t for t, _ in where} == {"above_right", "below_left", "corner", "above", "mrl2"}
    assert (recs["multiRefIdx"] == 2).any() and not (recs["y"][recs["multiRefIdx"] > 0] % ctu == 0).any()
    _rules_accept(case)
