"""Pins oracle/k2_inter.c against the reference at PU level: the real InterPrediction::motionCompensation (xPredInterBi/Uni,
xSubPuBio, xProcessDMVR, xPredAffineBlk incl. PROF, xWeightedAverage) runs on real CodingUnits and border-extended reference
Pictures built by the shim; predictions and DMVR MV deltas must match exactly."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth
from tests.helpers import ref_ptrs

pytestmark = pytest.mark.ref


def _case(seed, W, H, bd, **kw):
    rng = np.random.default_rng(seed)
    cus = synth.partition(rng, W, H)
    pus, ndmvr = synth.gen_pus(rng, cus, W, H, **kw)
    refs = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
    return pus, ndmvr, refs


def _compare(oracle, ref, simd, W, H, bd, pus, ndmvr, refs):
    g = abi.make_geom(W, H, bd)
    a = [np.full((H, W), -1, np.int16), np.full((H // 2, W // 2), -1, np.int16), np.full((H // 2, W // 2), -1, np.int16)]
    b = [p.copy() for p in a]
    da = np.zeros((ndmvr + 1, 2), np.int32); db = np.zeros((ndmvr + 1, 2), np.int32)
    rp = ref_ptrs(refs)
    oracle.orc_mc_predict(C.byref(g), abi.plane_ptrs(a), rp, pus.ctypes.data, len(pus), da.ctypes.data)
    rc = ref.ref_mc_predict(simd, C.byref(g), abi.plane_ptrs(b), rp, pus.ctypes.data, len(pus), db.ctypes.data, ndmvr)
    assert rc == 0, "the reference did not take the DMVR decision the PU flags ask for"
    for c in range(3):
        if not np.array_equal(a[c], b[c]):
            d = np.argwhere(a[c] != b[c]); y, x = d[0]; sh = 1 if c else 0
            hit = [i for i, p in enumerate(pus) if p["x"] >> sh <= x < (p["x"] + p["w"]) >> sh and p["y"] >> sh <= y < (p["y"] + p["h"]) >> sh]
            raise AssertionError(f"plane {c}: {len(d)} diffs, first at {(y, x)}: {a[c][y, x]} vs {b[c][y, x]}; PU {pus[hit[0]] if hit else None}")
    assert np.array_equal(da, db), f"DMVR deltas differ: {np.argwhere(da != db)[:5]}"
    return a


@pytest.mark.parametrize("simd", [0, 1])
def test_regular_uni_bi_bcw(oracle, ref, simd):
    pus, nd, refs = _case(1, 416, 240, 10, p_dmvr=0, p_bdof=0, p_affine=0)
    _compare(oracle, ref, simd, 416, 240, 10, pus, nd, refs)
    assert (pus["bcwW1"] != 4).any() and (pus["flags"] & synth.PU_ALTHPEL).any() and (pus["refSlot"][:, 1] < 0).any()


@pytest.mark.parametrize("simd", [0, 1])
def test_bdof(oracle, ref, simd):
    pus, nd, refs = _case(2, 416, 240, 10, p_dmvr=0, p_bdof=0.9, p_affine=0, p_bi=0.9)
    _compare(oracle, ref, simd, 416, 240, 10, pus, nd, refs)
    assert (pus["flags"] & synth.PU_BDOF).sum() > 20


@pytest.mark.parametrize("simd", [0, 1])
def test_dmvr(oracle, ref, simd):
    pus, nd, refs = _case(3, 416, 240, 10, p_dmvr=0.9, p_bdof=0.05, p_affine=0, p_bi=0.9, mv_sigma=2.0)
    _compare(oracle, ref, simd, 416, 240, 10, pus, nd, refs)
    assert (pus["flags"] & synth.PU_DMVR).sum() > 20


@pytest.mark.parametrize("simd", [0, 1])
def test_affine_prof(oracle, ref, simd):
    pus, nd, refs = _case(4, 416, 240, 10, p_dmvr=0, p_bdof=0, p_affine=0.9, p_prof=0.8)
    _compare(oracle, ref, simd, 416, 240, 10, pus, nd, refs)
    f = pus["flags"]
    assert (f & synth.PU_AFFINE).sum() > 20 and (f & synth.PU_AFFINE6).any() and (f & synth.PU_PROF0).any()


@pytest.mark.parametrize("seed,W,H,bd,simd", [(5, 1920, 1080, 10, 1), (6, 256, 128, 8, 0), (7, 384, 256, 12, 0)])
def test_mixed_pictures(oracle, ref, seed, W, H, bd, simd):
    # DMVR's 10-bit bilinear search is only defined for bit depths <= 10 in the reference (the >10-bit branch of filterCopy is
    # compiled out, InterpolationFilter.cpp:447-463), so the 12-bit case runs without DMVR.
    pus, nd, refs = _case(seed, W, H, bd, **({"p_dmvr": 0.0} if bd > 10 else {}))
    _compare(oracle, ref, simd, W, H, bd, pus, nd, refs)


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("bd", [8, 10])
def test_explicit_weighted_prediction(oracle, ref, simd, bd):
    """pps_weighted_bipred: the real xWeightedPredictionBi -> addWeightBi / addWeightUni (WeightPrediction.cpp) against the oracle's
    `weighted`, for uni, bi, BCW (which bypasses WP) and affine (+PROF) CUs; the b200_wp entries come from the generator's restatement
    of getWpScaling."""
    W, H = 256, 128
    for seed in (1, 2, 3):
        pus, ndmvr, refs = _case(seed * 7 + bd, W, H, bd, p_dmvr=0.0, p_bdof=0.0, p_affine=0.2, p_bcw=0.3)
        rng = np.random.default_rng(seed)
        raw, ent = synth.gen_wp(rng, bd, pus)
        assert (pus["wpIdx"] != 0).any() and (pus["wpIdx"] == 0).any()
        g = abi.make_geom(W, H, bd)
        a = [np.full((H, W), -1, np.int16), np.full((H // 2, W // 2), -1, np.int16), np.full((H // 2, W // 2), -1, np.int16)]
        b = [p.copy() for p in a]
        da = np.zeros((ndmvr + 1, 2), np.int32); db = np.zeros((ndmvr + 1, 2), np.int32)
        rp = ref_ptrs(refs)
        oracle.orc_mc_predict_wp(C.byref(g), abi.plane_ptrs(a), rp, pus.ctypes.data, len(pus), da.ctypes.data, ent.ctypes.data)
        ref.ref_set_wp(raw.ctypes.data)
        try:
            rc = ref.ref_mc_predict(simd, C.byref(g), abi.plane_ptrs(b), rp, pus.ctypes.data, len(pus), db.ctypes.data, ndmvr)
        finally:
            ref.ref_set_wp(None)
        assert rc == 0
        for c in range(3):
            assert np.array_equal(a[c], b[c]), f"plane {c}: {len(np.argwhere(a[c] != b[c]))} diffs"


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("bd", [8, 10])
def test_geo(oracle, ref, simd, bd):
    """Geometric partitioning: the real motionCompensationGeo (two uni-predictions + xWeightedGeoBlk) against the oracle's geo_blend with
    the dumped weight tables; all 64 split directions occur over the seeds, partitions from the same or different lists."""
    W, H = 384, 256
    seen = set()
    for seed in (1, 2, 3, 4):
        pus, ndmvr, refs = _case(seed * 3 + bd, W, H, bd, p_geo=0.6, p_dmvr=0.1, p_bdof=0.1)
        geo = pus[(pus["flags"] & 128) != 0]
        assert len(geo) > 30
        seen |= set(int(v) for v in geo["bcwW1"])
        _compare(oracle, ref, simd, W, H, bd, pus, ndmvr, refs)
    assert len(seen) >= 60


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("name", list(synth.MC_SWEEP_CASES))
def test_designed_sweep(oracle, ref, name, simd):
    """Every case of the designed K2 sweep (synth.mc_sweep: shapes x tools, phases, window thresholds at the picture edges, clipMv bounds for CTU 32 / 64
    / 128, MVs near +-2^17, affine spread limits, DMVR targets and designed cost surfaces; 8 / 10 / 12 bit, 4:0:0, padded and odd strides): the
    oracle and the real motion compensation give the same samples and DMVR deltas."""
    from tests.helpers import mc_dst, mc_oracle, mc_mismatch
    case = synth.mc_sweep(name)
    g, pus = case["g"], case["pus"]
    a, da = mc_oracle(oracle, case)
    b = mc_dst(g); db = np.zeros_like(da)
    if case["wp"]: ref.ref_set_wp(case["wp"][0].ctypes.data)
    try:
        rc = ref.ref_mc_predict(simd, C.byref(g), abi.plane_ptrs(b), ref_ptrs(case["refs"]), pus.ctypes.data, len(pus), db.ctypes.data, case["ndmvr"])
    finally:
        ref.ref_set_wp(None)
    assert rc == 0, "the reference did not take the DMVR decision the PU flags ask for"
    msg = mc_mismatch(case, a, b, da, db)
    assert msg is None, msg
