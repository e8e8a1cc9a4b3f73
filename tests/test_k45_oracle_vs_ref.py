"""Pins oracle/k4_sao.c and oracle/k5_alf.c against the reference: pointer level (offsetBlock, deriveClassificationBlk,
filter7x7Blk/5x5Blk, filterCcAlf) and picture level (real SAOProcessCTU / ALF prepareCTU+processCTU on a real CodingStructure)."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth
from tests.helpers import aligned

pytestmark = pytest.mark.ref


def _arr(a):
    return a.ctypes.data


@pytest.mark.parametrize("simd", [0, 1])
def test_sao_offset_block(oracle, ref, simd):
    rng = np.random.default_rng(1)
    for case in range(600):
        bd = int(rng.choice([8, 10, 12]))
        w = int(rng.choice([8, 16, 32, 64, 128, 24, 56])); h = int(rng.choice([8, 16, 32, 64, 128, 24, 56]))
        stride = w + 32
        base = aligned((h + 16, stride), np.int16)
        base[...] = (rng.integers(0, 1 << bd, size=base.shape) >> int(rng.integers(0, 5))) + (1 << (bd - 2))
        np.clip(base, 0, (1 << bd) - 1, out=base)
        t = case % 5
        offs = np.zeros(32, np.int32); band = 0
        if t == 4:
            band = int(rng.integers(0, 32))
            for i in range(4): offs[(band + i) & 31] = int(rng.integers(-31, 32))
        else:
            offs[:5] = rng.integers(-31, 32, size=5); offs[2] = 0
        avail = int(rng.integers(0, 256)) if case % 3 else 255
        if simd:
            # The SIMD path assumes a diagonal neighbour is only available when both adjacent ones are (always true for
            # raster slices / rectangular tiles); the scalar reference — our oracle's target — handles all 256 combinations.
            for d, (p, q) in {16: (1, 4), 32: (2, 4), 64: (1, 8), 128: (2, 8)}.items():
                if avail & d and not (avail & p and avail & q): avail &= ~d
            # ... and (raster order / rectangles) above-right and below-left can not be missing when both adjacent CTUs are there;
            # the reference's own scalar and SIMD disagree on exactly those impossible cases (EO_45 corner samples).
            if avail & 2 and avail & 4: avail |= 32
            if avail & 1 and avail & 8: avail |= 64
        nv = nh = 0; vv = np.zeros(3, np.int32); hh = np.zeros(3, np.int32)
        if case % 7 == 0:
            nv = int(rng.integers(0, 3)); nh = int(rng.integers(0, 3))
            vv[:nv] = np.sort(rng.choice(np.arange(8, w, 8), size=nv, replace=False)) if nv and w > 16 else 0
            hh[:nh] = np.sort(rng.choice(np.arange(8, h, 8), size=nh, replace=False)) if nh and h > 16 else 0
            if w <= 16: nv = 0
            if h <= 16: nh = 0
        o = 8 * stride + 16
        a = aligned(base.shape, np.int16); a[...] = base; b = aligned(base.shape, np.int16); b[...] = base
        oracle.orc_sao_offset_block(bd, t, _arr(offs), _arr(base) + 2 * o, _arr(a) + 2 * o, stride, stride, w, h, avail, nv, _arr(vv), nh, _arr(hh))
        ref.ref_sao_offset_block(simd, bd, t, _arr(offs), band, _arr(base) + 2 * o, _arr(b) + 2 * o, stride, stride, w, h, avail, nv, _arr(vv), nh, _arr(hh))
        assert np.array_equal(a, b), (case, t, w, h, avail, nv, nh, np.argwhere(a != b)[:5])


@pytest.mark.parametrize("seed,W,H,bd,ctu,simd,vb", [(1, 256, 128, 10, 128, 0, 0), (2, 416, 240, 10, 64, 1, 0), (3, 200, 136, 8, 32, 0, 1),
                                                    (4, 1920, 1080, 10, 128, 1, 0), (5, 384, 256, 12, 128, 0, 1)])
def test_sao_picture_vs_reference(oracle, ref, seed, W, H, bd, ctu, simd, vb):
    rng = np.random.default_rng(seed)
    src = synth.noise_planes(rng, W, H, bd)
    sao = synth.gen_sao(rng, W, H, ctu, bd, p_on=0.7)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    v = abi.Vb()
    if vb:
        v.numVer, v.numHor = 2, 1
        v.posX[0], v.posX[1], v.posY[0] = 8 * (W // 24), 8 * (W // 12), 8 * (H // 16)
    a = [np.zeros_like(p) for p in src]; b = [np.zeros_like(p) for p in src]
    oracle.orc_sao_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(a), _arr(sao), C.addressof(v))
    ref.ref_sao_picture(simd, C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(b), _arr(sao), C.addressof(v))
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c}: {np.argwhere(a[c] != b[c])[:8]}"
        assert not np.array_equal(a[c], src[c])


@pytest.mark.parametrize("simd", [0, 1])
def test_alf_classify(oracle, ref, simd):
    rng = np.random.default_rng(2)
    for case in range(120):
        bd = int(rng.choice([8, 10]))
        PW, PH = 96, 160
        plane = (rng.integers(0, 1 << bd, size=(PH, PW)) >> int(rng.integers(0, 4))).astype(np.int16)
        if case % 3 == 0:  # directional structure
            yy, xx = np.mgrid[0:PH, 0:PW]
            plane = ((np.sin((xx * (case % 5) + yy * (case % 7)) / 3.0) * 0.4 + 0.5) * ((1 << bd) - 1)).astype(np.int16)
        # reference view: padded by replication (prepareCTU); oracle view: same padded array, origin shifted
        pad = 8
        padded = np.pad(plane, pad, mode="edge")
        org = _arr(padded) + 2 * (pad * padded.shape[1] + pad)
        bx = int(rng.choice([0, 32, 64])); by = int(rng.choice([0, 32, 64, 96, 128])); bw = int(rng.choice([32, 32, 16, 8])); bh = int(rng.choice([32, 32, 24, 4]))
        a = np.zeros(64, np.uint16); b = np.zeros(64, np.uint16)
        oracle.orc_alf_classify(_arr(a), org, padded.shape[1], bx, by, bw, bh, bd + 4, 128, 124)
        ref.ref_alf_classify(simd, _arr(b), _arr(plane), PW, PW, PH, bx, by, bw, bh, bd + 4, 128, 124)
        m = np.zeros((8, 8), bool); m[:bh // 4, :bw // 4] = True
        assert np.array_equal(a.reshape(8, 8)[m], b.reshape(8, 8)[m]), (case, bx, by, bw, bh)


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("is7", [1, 0])
def test_alf_filter_blk(oracle, ref, simd, is7):
    rng = np.random.default_rng(3 + is7)
    for case in range(100):
        bd = 10
        PW, PH = 64, 160 if is7 else 96
        plane = (rng.integers(0, 1 << bd, size=(PH, PW)) >> int(rng.integers(0, 3))).astype(np.int16)
        pad = 8
        padded = np.pad(plane, pad, mode="edge")
        org = _arr(padded) + 2 * (pad * padded.shape[1] + pad)
        t = synth.gen_alf(rng, 128, 128, n_aps=1)
        cls = (rng.integers(0, 25, size=64) | (rng.integers(0, 4, size=64) << 8)).astype(np.uint16)
        vbH, vbPos = (128, 124) if is7 else (64, 62)
        bx = int(rng.choice([0, 32])); by = int(rng.choice(range(0, PH - 31, 32))); bw, bh = 32, 32
        a = plane.copy(); b = plane.copy()
        if is7:
            co, cl = t["lumaCoeff"][16], t["lumaClip"][16]
            oracle.orc_alf_filter_blk(1, _arr(cls), _arr(a), PW, org, padded.shape[1], bx, by, bw, bh, _arr(co), _arr(cl), bd, vbH, vbPos)
            ref.ref_alf_filter_blk(simd, 1, _arr(cls), _arr(b), PW, _arr(plane), PW, PW, PH, bx, by, bw, bh, _arr(co), _arr(cl), bd, vbH, vbPos)
        else:
            co, cl = t["chromaCoeff"][1], t["chromaClip"][1]
            oracle.orc_alf_filter_blk(0, None, _arr(a), PW, org, padded.shape[1], bx, by, bw, bh, _arr(co), _arr(cl), bd, vbH, vbPos)
            ref.ref_alf_filter_blk(simd, 0, None, _arr(b), PW, _arr(plane), PW, PW, PH, bx, by, bw, bh, _arr(co), _arr(cl), bd, vbH, vbPos)
        assert np.array_equal(a, b), (case, bx, by, np.argwhere(a != b)[:5])
        assert not np.array_equal(a, plane)


@pytest.mark.parametrize("simd", [0, 1])
def test_alf_ccalf_blk(oracle, ref, simd):
    rng = np.random.default_rng(5)
    for case in range(100):
        bd = int(rng.choice([8, 10]))
        LW, LH = 128, 256
        luma = (rng.integers(0, 1 << bd, size=(LH, LW)) >> int(rng.integers(0, 3))).astype(np.int16)
        pad = 8
        padded = np.pad(luma, pad, mode="edge")
        org = _arr(padded) + 2 * (pad * padded.shape[1] + pad)
        chroma = rng.integers(0, 1 << bd, size=(LH // 2, LW // 2)).astype(np.int16)
        f = rng.integers(-63, 64, size=7).astype(np.int16)
        cx, cy, cw, ch = int(rng.choice([0, 32])), int(rng.choice([0, 64])), 32, 64
        a = chroma.copy(); b = chroma.copy()
        oracle.orc_alf_ccalf_blk(_arr(a), LW // 2, org, padded.shape[1], cx, cy, cw, ch, _arr(f), bd, 128, 124)
        ref.ref_alf_ccalf_blk(simd, _arr(b), LW // 2, _arr(luma), LW, LW, LH, cx, cy, cw, ch, _arr(f), bd, 128, 124)
        assert np.array_equal(a, b), (case, np.argwhere(a != b)[:5])


@pytest.mark.parametrize("seed,W,H,bd,ctu,simd", [(1, 256, 128, 10, 128, 0), (2, 416, 240, 10, 64, 1), (3, 200, 136, 8, 32, 0),
                                                 (4, 1920, 1080, 10, 128, 1), (5, 384, 256, 10, 128, 0)])
def test_alf_picture_vs_reference(oracle, ref, seed, W, H, bd, ctu, simd):
    rng = np.random.default_rng(seed)
    src = synth.noise_planes(rng, W, H, bd)
    t = synth.gen_alf(rng, W, H, ctu, bd, n_aps=3)
    T = abi.make_alf_tables(t)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    a = [np.zeros_like(p) for p in src]; b = [np.zeros_like(p) for p in src]
    oracle.orc_alf_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(a), _arr(t["ctus"]), C.byref(T))
    ref.ref_alf_picture(simd, C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(b), _arr(t["ctus"]), C.byref(T))
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c}: {len(np.argwhere(a[c] != b[c]))} diffs, first {np.argwhere(a[c] != b[c])[:8]}"
        assert not np.array_equal(a[c], src[c])


def _width(planes, case):
    return [p[:, :(case["W"] >> (c > 0))] for c, p in enumerate(planes)]


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("name", [n for n in synth.SAO_SWEEP_CASES if n != "avail_masks_ctu32"])
def test_sao_sweep_vs_reference(oracle, ref, name, simd):
    """Every case of the designed SAO sweep with the picture's own CTU availability (the reference derives it from the picture) equals the real
    SAOProcessCTU: every band start, the largest offsets at 8 / 9 / 10 / 12 bit, every EO category, 0..3 virtual boundaries per direction, partial CTUs,
    4:0:0, padded strides and 4K."""
    case = synth.sao_sweep(name)
    a = [np.zeros_like(p) for p in case["planes"]]; b = [np.zeros_like(p) for p in case["planes"]]
    oracle.orc_sao_picture(C.byref(case["g"]), abi.plane_ptrs(case["planes"]), abi.plane_ptrs(a), _arr(case["ctus"]), C.addressof(case["vb"]))
    ref.ref_sao_picture(simd, C.byref(case["g"]), abi.plane_ptrs(case["planes"]), abi.plane_ptrs(b), _arr(case["ctus"]), C.addressof(case["vb"]))
    for c, (x, y) in enumerate(zip(_width(a, case), _width(b, case))):
        assert np.array_equal(x, y), f"{name}: plane {c}: {np.argwhere(x != y)[:8]}"


def test_sao_sweep_avail_masks_vs_reference(oracle, ref):
    """The 256-mask case, CTU by CTU through offsetBlock with each CTU's own mask (the picture-level reference derives availability itself).  Scalar only:
    the reference's SIMD path assumes masks that raster slices and rectangular tiles can produce, and disagrees with its scalar code on the others (see
    test_sao_offset_block)."""
    case = synth.sao_sweep("avail_masks_ctu32")
    ctu, W = case["ctu"], case["W"]
    ctusW, ctusH = (W + ctu - 1) // ctu, (case["H"] + ctu - 1) // ctu
    for i, r in enumerate(case["ctus"]):
        cx, cy = i % ctusW, i // ctusW
        if not (0 < cx < ctusW - 1 and 0 < cy < ctusH - 1): continue
        for c in range(3):
            t = int(r["type"][c])
            if t == 255: continue
            sh = 1 if c else 0
            p = case["planes"][c]; stride = p.shape[1]
            offs = np.zeros(32, np.int32); band = int(r["band"][c])
            if t == 4:
                for k in range(4): offs[(band + k) & 31] = r["offset"][c][k]
            else: offs[:5] = r["offset"][c]
            o = ((cy * ctu) >> sh) * stride + ((cx * ctu) >> sh)
            a = p.copy(); b = p.copy(); nv = np.zeros(3, np.int32)
            oracle.orc_sao_offset_block(case["bd"], t, _arr(offs), _arr(p) + 2 * o, _arr(a) + 2 * o, stride, stride, ctu >> sh, ctu >> sh, int(r["avail"]), 0, _arr(nv), 0, _arr(nv))
            ref.ref_sao_offset_block(0, case["bd"], t, _arr(offs), band, _arr(p) + 2 * o, _arr(b) + 2 * o, stride, stride, ctu >> sh, ctu >> sh, int(r["avail"]), 0, _arr(nv), 0, _arr(nv))
            assert np.array_equal(a, b), (i, c, t, int(r["avail"]), np.argwhere(a != b)[:4])


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("name", [n for n in synth.ALF_SWEEP_CASES if not synth.alf_sweep(n)["flagged"]])
def test_alf_sweep_vs_reference(oracle, ref, name, simd):
    """Every case of the designed ALF sweep without clip / pad flags equals the real ALF prepareCTU + processCTU: every class x transpose, the scalar
    path, int8 extremes, every clip index, every CC-ALF coefficient, chromaAlt 0..7, 8 / 9 / 10 bit, CTU 32 / 64 / 128, 4:0:0, padded strides and 4K.
    The flagged cases are pinned through the seam (slices with loop filtering across them disabled, tests/test_seam_cpu.py)."""
    case = synth.alf_sweep(name)
    t = case["tables"]
    T = abi.make_alf_tables(t)
    a = [np.zeros_like(p) for p in case["planes"]]; b = [np.zeros_like(p) for p in case["planes"]]
    oracle.orc_alf_picture(C.byref(case["g"]), abi.plane_ptrs(case["planes"]), abi.plane_ptrs(a), _arr(t["ctus"]), C.byref(T))
    ref.ref_alf_picture(simd, C.byref(case["g"]), abi.plane_ptrs(case["planes"]), abi.plane_ptrs(b), _arr(t["ctus"]), C.byref(T))
    for c, (x, y) in enumerate(zip(_width(a, case), _width(b, case))):
        assert np.array_equal(x, y), f"{name}: plane {c}: {len(np.argwhere(x != y))} diffs, first {np.argwhere(x != y)[:8]}"
