"""LMCS: the oracle's restatement (oracle/k6_lmcs.c) and the generator's table construction against the reference's real Reshape class
and PelBufferOps pointers (scalar and SIMD), function level and picture level."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth
from tests.helpers import aligned, aligned_copy, ref_ptrs, oracle_decompress

pytestmark = pytest.mark.ref


def build(ref, rng, bd, chroma_adj=True):
    """random legal model -> (Lmcs from the REAL constructReshaper, generator's dict)"""
    cus = np.array([[0, 0, 64, 64]])
    m = synth.gen_lmcs(rng, bd, cus, 64, 64, 64, chroma_adj=chroma_adj)
    L = abi.Lmcs(); lut = np.zeros(1 << bd, np.int16)
    delta = (C.c_int * 16)(*m["delta"])
    assert ref.ref_lmcs_build(bd, m["minBin"], m["maxBin"], delta, m["chrOff"], int(chroma_adj), C.byref(L), lut) == 0
    return L, lut, m


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_tables_match_construct_reshaper(ref, bd):
    rng = np.random.default_rng(bd)
    for _ in range(20):
        L, lut, m = build(ref, rng, bd)
        G = m["struct"]
        assert (L.orgCW, L.minBinIdx, L.maxBinIdx) == (G.orgCW, G.minBinIdx, G.maxBinIdx)
        assert list(L.reshapePivot) == list(G.reshapePivot) and list(L.inputPivot) == list(G.inputPivot)
        assert list(L.fwdScaleCoef) == list(G.fwdScaleCoef) and list(L.chromaAdjHelpLUT) == list(G.chromaAdjHelpLUT)
        assert np.array_equal(lut, m["invLUT"])


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_forward_inverse_scale(oracle, ref, bd, simd):
    rng = np.random.default_rng(100 + bd + simd)
    for (w, h) in [(4, 4), (8, 4), (16, 16), (64, 32), (128, 128), (4, 64)]:
        L, lut, m = build(ref, rng, bd)
        st = (w + 15) // 16 * 16 + 16                                # the AVX2 paths use aligned 32-byte row loads (picture buffers are)
        src = rng.integers(0, 1 << bd, size=(h, st)).astype(np.int16); src[0, :4] = [0, (1 << bd) - 1, 1, (1 << bd) - 2]
        a = aligned_copy(src); b = aligned_copy(src)
        ref.ref_lmcs_fwd_block(simd, a.ctypes.data, st, w, h)
        oracle.orc_lmcs_fwd_block(b.ctypes.data, st, w, h, bd, C.byref(L))
        assert np.array_equal(a, b), ("fwd", w, h)
        a = aligned_copy(src); b = aligned_copy(src)
        ref.ref_lmcs_inv_block(simd, a.ctypes.data, st, w, h)          # SIMD: the piece-wise linear rspBcw; scalar: applyLut(m_invLUT)
        b[:, :w] = lut[b[:, :w]]
        assert np.array_equal(a, b), ("inv", w, h)
        # scaleSignal: residuals incl. the extremes, every LUT entry
        res = rng.integers(-(1 << bd) - 40, (1 << bd) + 40, size=(h, w)).astype(np.int16); res[0, :2] = [-32768, 32767]
        for sc in sorted(set(L.chromaAdjHelpLUT)):
            a = res.copy()
            ref.ref_lmcs_scale_block(a.ctypes.data, w, w, h, sc, bd)
            want = np.array([oracle.orc_lmcs_scale_resi(int(v), sc, bd) for v in res.reshape(-1)], np.int16).reshape(h, w)
            assert np.array_equal(a, want), ("scale", sc)


@pytest.mark.parametrize("ctu,W,H", [(128, 256, 192), (64, 192, 136), (32, 96, 72)])
def test_vpdu_chroma_scale(oracle, ref, ctu, W, H):
    """calculateChromaAdjVpduNei on a picture with one CU per CTU: every VPDU, incl. the picture-edge clamps of the neighbour walk."""
    bd = 10
    rng = np.random.default_rng(ctu)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    L, lut, m = build(ref, rng, bd)
    planes = synth.noise_planes(rng, W, H, bd)
    vs = 64 if ctu == 128 else ctu
    for vy in range(0, H, vs):
        for vx in range(0, W, vs):
            cx, cy = vx // ctu * ctu, vy // ctu * ctu          # the CU covering the VPDU's top-left = its CTU
            v = abi.LmcsVpdu(cx, cy, int(cx > 0), int(cy > 0))
            want = ref.ref_lmcs_vpdu_scale(C.byref(g), abi.plane_ptrs(planes), vx, vy)
            got = oracle.orc_lmcs_vpdu_scale(C.byref(g), planes[0], C.byref(L), C.byref(v))
            assert got == want, (vx, vy)


def build_model(ref, name, bd):
    """designed model -> (Lmcs from the REAL constructReshaper, its invLUT, the generator's dict)"""
    m = synth.lmcs_model(name, bd)
    L = abi.Lmcs(); lut = np.zeros(1 << bd, np.int16)
    assert ref.ref_lmcs_build(bd, m["minBin"], m["maxBin"], (C.c_int * 16)(*m["delta"]), m["chrOff"], 1, C.byref(L), lut) == 0, name
    return L, lut, m


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_designed_models_match_construct_reshaper(oracle, ref, bd):
    """Every designed model (synth.LMCS_MODELS): constructReshaper accepts it and builds lmcs_tables' tables; rspBufFwd / applyLut on a ramp of every
    value equal the oracle's forward map and the LUT (scalar and SIMD).  The SIMD inverse (rspBcw, piece-wise linear) agrees with the LUT on every
    designed model."""
    n = 1 << bd
    for name in synth.LMCS_MODELS:
        L, lut, m = build_model(ref, name, bd)
        G = m["struct"]
        assert (L.orgCW, L.minBinIdx, L.maxBinIdx) == (G.orgCW, G.minBinIdx, G.maxBinIdx), name
        assert list(L.reshapePivot) == list(G.reshapePivot) and list(L.inputPivot) == list(G.inputPivot), name
        assert list(L.fwdScaleCoef) == list(G.fwdScaleCoef) and list(L.chromaAdjHelpLUT) == list(G.chromaAdjHelpLUT), name
        assert np.array_equal(lut, m["invLUT"]), name
        st = 64
        ramp = np.arange(((n + st - 1) // st) * st).reshape(-1, st).astype(np.int16) % n
        for simd in (0, 1):
            a = aligned_copy(ramp); b = aligned_copy(ramp)
            ref.ref_lmcs_fwd_block(simd, a.ctypes.data, st, st, len(ramp))
            oracle.orc_lmcs_fwd_block(b.ctypes.data, st, st, len(ramp), bd, C.byref(L))
            assert np.array_equal(a, b), ("fwd", name, simd)
            a = aligned_copy(ramp)
            ref.ref_lmcs_inv_block(simd, a.ctypes.data, st, st, len(ramp))
            assert np.array_equal(a, lut[ramp]), ("inv", name, simd, int((a != lut[ramp]).sum()))


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_designed_vpdu_neighbourhoods(oracle, ref, bd):
    """calculateChromaAdjVpduNei on the sweep's designed neighbourhoods (one CU per CTU at CTU 32 and 64, as the shim's structure; averages on every
    pivot, walks clamped at the picture's last row / column) equals orc_lmcs_vpdu_scale for every VPDU."""
    for var in ("ctu32", "ctu64"):
        name = [k for k in synth.LMCS_SWEEP if k.startswith("vpdu_") and k.endswith(f"_{bd}bit_{var}")][0]
        c = synth.lmcs_sweep(name)
        m = c["pic"]["lmcs"]
        L, lut, _ = build_model(ref, m["name"], bd)
        vs = min(64, c["ctu"]); vW = (c["W"] + vs - 1) // vs
        planes = [c["pic"]["given"][0], np.zeros((c["H"] // 2, c["W"] // 2), np.int16), np.zeros((c["H"] // 2, c["W"] // 2), np.int16)]
        for i, v in enumerate(m["vpdus"]):
            want = ref.ref_lmcs_vpdu_scale(C.byref(c["g"]), abi.plane_ptrs(planes), (i % vW) * vs, (i // vW) * vs)
            vv = abi.LmcsVpdu(int(v["x"]), int(v["y"]), int(v["availLeft"]), int(v["availAbove"]))
            assert oracle.orc_lmcs_vpdu_scale(C.byref(c["g"]), planes[0], C.byref(m["struct"]), C.byref(vv)) == want, (name, i)


@pytest.mark.parametrize("name", ["vpdu_full_bins_8bit_ctu32", "vpdu_full_bins_10bit_ctu32", "vpdu_full_bins_12bit_ctu32", "extremes_crs_min_12bit"])
def test_sweep_pictures_reference_arm(oracle, ref, name):
    """The reference arm (ref_decompress_picture_out, SIMD off) equals oracle_decompress on sweep pictures whose records are CTU origins."""
    c = synth.lmcs_sweep(name)
    want, _ = oracle_decompress(oracle, c["g"], c["dpb"], c["pic"])
    got = [np.zeros_like(p) for p in want]
    ref.ref_decompress_picture_out(C.byref(c["g"]), ref_ptrs(c["dpb"]), C.byref(c["pic"]["struct"]), 2, 0, abi.plane_ptrs(got))
    for k in range(3):
        assert np.array_equal(want[k], got[k]), (name, k, int((want[k] != got[k]).sum()))


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("chroma_adj", [True, False])
def test_picture_with_lmcs(oracle, ref, simd, chroma_adj):
    """Whole back end with LMCS on: oracle chain vs the reference's kernels (real rspBufFwd / calculateChromaAdjVpduNei / scaleSignal /
    rspBcw|applyLut inside the multi-threaded reference arm).  The reference arm's structure has one CU per CTU, so the VPDU records
    point at CTU origins here."""
    W, H, bd, ctu = 256, 192, 10, 128
    rng = np.random.default_rng(7 + simd)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    dpb = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
    pic = synth.gen_picture(rng, W, H, bd, dst_slot=0, lmcs=True, lmcs_chroma=chroma_adj)
    vp = pic["lmcs"]["vpdus"]
    for j in range((H + 63) // 64):
        for i in range((W + 63) // 64):
            cx, cy = i * 64 // ctu * ctu, j * 64 // ctu * ctu
            vp[j * ((W + 63) // 64) + i] = (cx, cy, cx > 0, cy > 0)
    want, _ = oracle_decompress(oracle, g, dpb, pic)
    got = [np.zeros_like(p) for p in want]
    ref.ref_decompress_picture_out(C.byref(g), ref_ptrs(dpb), C.byref(pic["struct"]), 3, simd, abi.plane_ptrs(got))
    for c in range(3):
        assert np.array_equal(want[c], got[c]), f"plane {c}: {len(np.argwhere(want[c] != got[c]))} diffs"
