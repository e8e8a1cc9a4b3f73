"""The designed LMCS sweep (synth.lmcs_model / synth.lmcs_sweep) reaches what tests/test_lmcs_gpu.py claims: legal models, ramps of every value, VPDU
neighbour averages on every pivot of the model, every availability, the picture-edge clamps, CUs over several VPDUs, the clip16 bound of the chroma
residual scaling at 12 bit and both paths of the inverse-map kernel.  No device and no reference needed (the C oracle only)."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth

BDS = (8, 10, 12)
SWEEP = synth.LMCS_SWEEP


def cases(kind, bd=None):
    return [n for n, (k, m, b, v) in SWEEP.items() if k == kind and (bd is None or b == bd)]


@pytest.mark.parametrize("bd", BDS)
def test_models_are_legal(bd):
    """Every designed model passes constructReshaper's conformance checks, and its tables are lmcs_tables' (so the device sees a model the reference
    would have built)."""
    org, step = (1 << bd) // 16, 1 << (bd - 5)
    for name in synth.LMCS_MODELS:
        m = synth.lmcs_model(name, bd)
        assert synth.lmcs_model_problems(bd, m["minBin"], m["maxBin"], m["delta"], m["chrOff"]) == [], name
        cw = [m["delta"][i] + org for i in range(m["minBin"], m["maxBin"] + 1)]
        t = m["tables"]
        if name == "identity": assert set(m["delta"]) == {0}
        if name == "compress": assert max(cw) <= org
        if name == "expand_max": assert (org << 3) - 1 in cw and (org >> 3) in cw
        if name == "fine_pivots":
            assert sum(c % step != 0 for c in cw) >= len(cw) // 2 and any(p % step for p in t["reshapePivot"][1:16])
        if name == "narrow_bins": assert (m["minBin"], m["maxBin"]) == (5, 9)
        if name == "single_bin": assert m["minBin"] == m["maxBin"]
        if name == "full_bins": assert (m["minBin"], m["maxBin"]) == (0, 15)
        if name == "crs_min": assert m["chrOff"] == -7 and min(cw) - 7 == org >> 3 and 16384 in t["chromaAdjHelpLUT"]
        if name == "crs_max": assert m["chrOff"] == 7 and max(cw) + 7 == (org << 3) - 1
    # an inverse coefficient at its largest (OrgCW / (OrgCW >> 3) = 8) and a forward slope near 8x
    e = synth.lmcs_model("expand_max", bd)["tables"]
    assert max(e["fwdScaleCoef"]) >= 8 * 2048 - 2048 // org - 1
    assert synth.lmcs_model_problems(bd, 0, 15, [0] * 16, 0), "all 16 bins at OrgCW break the sum rule"


@pytest.mark.parametrize("bd", BDS)
def test_forward_map_never_needs_its_clip(bd):
    """On a legal model the forward map of every value stays inside 0 .. 2^bd - 1 before its clip (a bin maps to at most its own code words), so the
    clip in lmcs_fwd never binds: expand_max brings the unclipped value closest to the top of its bins."""
    pmax = (1 << bd) - 1
    for name in synth.LMCS_MODELS:
        m = synth.lmcs_model(name, bd)
        f = synth.lmcs_fwd(m, np.arange(pmax + 1))
        assert f.min() >= 0 and f.max() <= pmax, name
        assert f.max() <= m["tables"]["reshapePivot"][16], name


@pytest.mark.parametrize("bd", BDS)
def test_compress_inverse_is_injective_on_the_forward_range(bd):
    """Under compress the inverse LUT is strictly increasing on pivot[minBin] .. pivot[maxBin + 1] - 1, which holds every forward value: a forward value
    off by one changes the picture after the inverse map, so the forward cases cannot hide a wrong K2 store."""
    m = synth.lmcs_model("compress", bd)
    t = m["tables"]; lut = t["invLUT"].astype(np.int64)
    lo, hi = t["reshapePivot"][m["minBin"]], t["reshapePivot"][m["maxBin"] + 1]
    assert (np.diff(lut[lo:hi]) > 0).all()
    f = synth.lmcs_fwd(m, np.arange(1 << bd))
    assert f.min() >= lo and f.max() < hi
    assert len(np.unique(lut[f])) == len(np.unique(f))


@pytest.mark.parametrize("bd", BDS)
def test_ramps_hold_every_value(bd):
    for name in cases("inverse", bd):
        c = synth.lmcs_sweep(name)
        y = c["pic"]["given"][0][:, :c["W"]]
        assert set(np.unique(y).tolist()) == set(range(1 << bd)), name
        assert (c["pic"]["given"][0][:, c["W"]:] == -7).all()
    for name in cases("forward", bd):
        c = synth.lmcs_sweep(name)
        assert set(np.unique(c["dpb"][0][0]).tolist()) == set(range(1 << bd)), name
        pus = c["pic"]["pus"]
        cover = np.zeros((c["H"], c["W"]), np.int32)
        for p in pus: cover[p["y"]:p["y"] + p["h"], p["x"]:p["x"] + p["w"]] += 1
        assert (cover == 1).all(), name                               # every sample predicted exactly once
        assert ((pus["refSlot"][:, 0] == 0) & (pus["refSlot"][:, 1] == 0)).sum() == 1 and (pus["mv"] == 0).all() and (pus["flags"] == 0).all()
        assert len({(int(p["w"]), int(p["h"])) for p in pus}) >= 4


def test_inverse_cases_reach_both_kernel_paths():
    """lmcs_inv_kernel stores 8 samples as one 16-byte word where the luma stride is a multiple of 8, sample by sample elsewhere."""
    for bd in BDS:
        for m in synth.LMCS_MODELS:
            assert synth.lmcs_sweep(f"inverse_{m}_{bd}bit_stride8")["g"].stride[0] % 8 == 0
            assert synth.lmcs_sweep(f"inverse_{m}_{bd}bit_odd")["g"].stride[0] % 2 == 1


def _averages(c):
    g, vp = c["g"], c["pic"]["lmcs"]["vpdus"]
    luma = c["pic"]["given"][0]
    return [synth.lmcs_average(luma, v, c["W"], c["H"], c["ctu"], c["bd"]) for v in vp]


@pytest.mark.parametrize("bd", BDS)
def test_vpdu_averages_hit_every_pivot(oracle, bd):
    """The VPDU neighbour averages land on pivot - 1, pivot and pivot + 1 of every bin boundary of the model, on 0 and on 2^bd - 1 (above maxBin's
    pivot: with maxBin 15, getPWLIdxInv's min(idx, 15)); the oracle's per-VPDU scale agrees with the average's bin."""
    for name in [n for n in cases("vpdu", bd) if not n.endswith("ctu128")]:
        c = synth.lmcs_sweep(name)
        m = c["pic"]["lmcs"]
        got = set(_averages(c))
        missing = set(synth.lmcs_targets(m, bd)) - got
        assert not missing, (name, sorted(missing))
        scale = np.zeros(len(m["vpdus"]), np.int32)
        oracle.orc_lmcs_vpdu_scales(C.byref(c["g"]), c["pic"]["given"][0], C.byref(m["struct"]), scale.ctypes.data)
        piv, lut = m["tables"]["reshapePivot"], m["tables"]["chromaAdjHelpLUT"]
        bins = set()
        for v, avg, s in zip(m["vpdus"], _averages(c), scale.tolist()):
            idx = m["minBin"]
            while idx <= m["maxBin"] and not avg < piv[idx + 1]: idx += 1
            bins.add(idx)
            assert s == lut[min(idx, 15)], (name, v, avg)
        assert bins >= set(range(m["minBin"], m["maxBin"] + 2)), (name, bins)   # every bin, and past maxBin
    m = synth.lmcs_sweep(f"vpdu_full_bins_{bd}bit_ctu32")["pic"]["lmcs"]
    assert m["maxBin"] == 15 and (1 << bd) - 1 >= m["tables"]["reshapePivot"][16]


@pytest.mark.parametrize("bd", BDS)
def test_vpdu_records_cover_availability_clamps_and_shared_cus(bd):
    """Every availability (none, left, above, both) occurs; the walks of some records reach past the picture's last row and last column (the clamps of
    lmcs_vpdu_kernel); some CUs cover several VPDUs (CTU 128: a 128x128 and 64x128 CUs); CTU 32, 64 and 128 give walks of 32 and 64 samples."""
    avail, clampH, clampW, shared, walks = set(), False, False, False, set()
    for name in cases("vpdu", bd):
        c = synth.lmcs_sweep(name)
        vp = c["pic"]["lmcs"]["vpdus"]; nn = min(64, c["ctu"])
        walks.add(nn)
        for v in vp:
            avail.add((int(v["availLeft"]), int(v["availAbove"])))
            clampH |= bool(v["availLeft"]) and int(v["y"]) + nn > c["H"]
            clampW |= bool(v["availAbove"]) and int(v["x"]) + nn > c["W"]
        origins = [(int(v["x"]), int(v["y"])) for v in vp]
        shared |= len(set(origins)) < len(origins)
        assert c["W"] % 64 or c["H"] % 64 or c["ctu"] == 32, name
    assert avail == {(0, 0), (1, 0), (0, 1), (1, 1)} and clampH and clampW and shared and walks == {32, 64}


@pytest.mark.parametrize("bd", BDS)
def test_vpdu_chroma_tus(bd):
    """One DC chroma TU per VPDU in Cb and in Cr, 4-sample chroma TUs (never scaled) and joint CbCr in every VPDU case."""
    for name in cases("vpdu", bd):
        c = synth.lmcs_sweep(name)
        tus = c["pic"]["tus"]
        n = len(c["pic"]["lmcs"]["vpdus"])
        assert sum("DC" in t and "Cb" in t for t in c["tags"]) == n and sum("DC" in t and "Cr" in t for t in c["tags"]) == n
        assert ((tus["log2w"] + tus["log2h"]) == 2).any() and (tus["ict"] != 0).any(), name


def test_12bit_scaled_residual_reaches_clip16(oracle):
    """At 12 bit under crs_min (chroma scale 16384) a residual of -2^bd scales to -4096 * 16384 >> 11 = -32768, the bound of clip16 in lmcs_scale; the
    extremes case carries such TUs in VPDUs whose neighbour averages select the 16384 bins."""
    c = synth.lmcs_sweep("extremes_crs_min_12bit")
    m = c["pic"]["lmcs"]
    scale = np.zeros(len(m["vpdus"]), np.int32)
    oracle.orc_lmcs_vpdu_scales(C.byref(c["g"]), c["pic"]["given"][0], C.byref(m["struct"]), scale.ctypes.data)
    hit = False
    tus, coefs = c["pic"]["tus"], c["pic"]["coefs"]
    vs = 64 if c["ctu"] == 128 else c["ctu"]; vW = (c["W"] + vs - 1) // vs
    for t in tus:
        w, h = 1 << int(t["log2w"]), 1 << int(t["log2h"])
        if w * h <= 4: continue
        r = np.zeros(w * h, np.int16)
        oracle.orc_tu_residual(C.byref(abi.Tu.from_buffer_copy(t.tobytes())), 12, coefs, None, r, w)
        sc = int(scale[((int(t["y"]) * 2) // vs) * vW + (int(t["x"]) * 2) // vs])
        hit |= any(oracle.orc_lmcs_scale_resi(int(v), sc, 12) == -32768 for v in set(r.tolist()))
    assert hit and (scale == 16384).any()


def test_yuv400_cases():
    for bd in BDS:
        on, off = synth.lmcs_sweep(f"yuv400_fine_pivots_{bd}bit_adj"), synth.lmcs_sweep(f"yuv400_fine_pivots_{bd}bit_noadj")
        assert on["g"].chromaFormat == 0 and on["pic"]["lmcs"]["struct"].chromaAdj == 1 and off["pic"]["lmcs"]["struct"].chromaAdj == 0
        assert len(on["pic"]["tus"]) and (on["pic"]["tus"]["comp"] == 0).all()
