"""Pins oracle/k3_deblock.c against the reference: pointer level (xPelFilterLuma, xFilteringPandQ — the latter is
not covered by the reference's own unit test) and picture level (the real LoopFilter::loopFilterCTU on a real
vvdec CodingStructure carrying our synthetic planes + LoopFilterParam grids)."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth
from tests.helpers import aligned

pytestmark = pytest.mark.ref


def _ptr(a, off):
    return a.ctypes.data + 2 * off


@pytest.mark.parametrize("simd", [0, 1])
def test_pel_filter_luma(oracle, ref, simd):
    rng = np.random.default_rng(1)
    for case in range(400):
        bd = int(rng.choice([8, 10, 12]))
        base = rng.integers(0, 1 << bd, size=(16, 32)).astype(np.int16)
        if case % 3: base = (base // 32 + (1 << (bd - 1))).astype(np.int16)      # smooth -> filters actually trigger
        a = aligned(base.shape, np.int16); a[...] = base; b = aligned(base.shape, np.int16); b[...] = base
        ver = case & 1
        off, step = (1, 32) if ver else (32, 1)
        o = 8 * 32 + 8
        args = (int(rng.integers(0, 30)), int(rng.integers(0, 2)), int(rng.integers(0, 300)), int(rng.integers(0, 2)), int(rng.integers(0, 2)), bd)
        oracle.orc_lf_pel_filter_luma(_ptr(a, o), step, off, *args)
        ref.ref_lf_pel_filter_luma(simd, _ptr(b, o), step, off, *args)
        assert np.array_equal(a, b), (case, args)


@pytest.mark.parametrize("simd", [0, 1])
def test_filtering_pq(oracle, ref, simd):
    rng = np.random.default_rng(2)
    for case in range(400):
        base = (rng.integers(0, 64, size=(24, 32)) + 400).astype(np.int16) if case % 2 else rng.integers(0, 1024, size=(24, 32)).astype(np.int16)
        a = aligned(base.shape, np.int16); a[...] = base; b = aligned(base.shape, np.int16); b[...] = base
        ver = case & 1
        off, step = (1, 32) if ver else (32, 1)
        o = 12 * 32 + 12
        nP, nQ = [(7, 7), (7, 5), (5, 7), (7, 3), (3, 7), (5, 5), (5, 3), (3, 5)][case % 8]
        tc = int(rng.integers(0, 40))
        oracle.orc_lf_filtering_pq(_ptr(a, o), step, off, nP, nQ, tc)
        ref.ref_lf_filtering_pq(simd, _ptr(b, o), step, off, nP, nQ, tc)
        assert np.array_equal(a, b), (case, nP, nQ, tc)


def _picture_case(rng, W, H, bd, ctu, nslices=1, ladf=False):
    cus = synth.partition(rng, W, H, ctu=ctu)
    lfV, lfH = synth.gen_lf_grid(rng, cus, W, H, bd)
    planes = synth.noise_planes(rng, W, H, bd)
    sl = np.zeros(nslices, synth.LFSLICE_DTYPE)
    sl["beta"] = rng.integers(-4, 5, size=(nslices, 3)); sl["tc"] = rng.integers(-4, 5, size=(nslices, 3))
    if nslices > 2: sl["disable"][1] = 1
    nctu = ((W + ctu - 1) // ctu) * ((H + ctu - 1) // ctu)
    ctu_slice = np.sort(rng.integers(0, nslices, size=nctu)).astype(np.uint8)
    seq = abi.LfSeq()
    if ladf:
        seq.ladfEnabled, seq.ladfNumIntervals = 1, 3
        for k, (o, b) in enumerate([(1, 0), (-2, 300), (3, 700)]): seq.ladfQpOffset[k] = o; seq.ladfIntervalLowerBound[k] = b
    return cus, lfV, lfH, planes, sl, ctu_slice, seq


@pytest.mark.parametrize("seed,W,H,bd,ctu,nsl,ladf,simd", [(1, 256, 128, 10, 128, 1, 0, 0), (2, 416, 240, 10, 64, 2, 1, 0),
                                                          (3, 200, 136, 8, 32, 3, 0, 1), (4, 1920, 1080, 10, 128, 1, 0, 1),
                                                          (5, 384, 256, 12, 128, 1, 1, 0)])
def test_deblock_picture_vs_reference(oracle, ref, seed, W, H, bd, ctu, nsl, ladf, simd):
    rng = np.random.default_rng(seed)
    cus, lfV, lfH, planes, sl, ctu_slice, seq = _picture_case(rng, W, H, bd, ctu, nsl, ladf)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    a = [p.copy() for p in planes]; b = [p.copy() for p in planes]
    oracle.orc_lf_deblock(C.byref(g), abi.plane_ptrs(a), lfV.ctypes.data, lfH.ctypes.data, ctu_slice.ctypes.data,
                          sl.ctypes.data, C.addressof(seq), 3)
    ref.ref_lf_deblock_picture(simd, C.byref(g), abi.plane_ptrs(b), lfV.ctypes.data, lfH.ctypes.data, ctu_slice.ctypes.data,
                               sl.ctypes.data, nsl, C.addressof(seq), 3)
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c}: {np.argwhere(a[c] != b[c])[:8]}"
        assert not np.array_equal(a[c], planes[c]), "deblocking changed nothing — test content too weak"
    # long filters must have been exercised
    assert ((lfV["len"] >> 4) & 7 == 7).any()


@pytest.mark.parametrize("simd", [0, 1])
@pytest.mark.parametrize("name", list(synth.LF_SWEEP_CASES))
def test_deblock_sweep_vs_reference(oracle, ref, name, simd):
    """Every case of the designed sweep (synth.lf_sweep) through the real LoopFilter, 4:0:0 and 64 slices included: the oracle's planes equal the
    reference's, stride padding included."""
    from tests.helpers import lf_args, lf_oracle, lf_mismatch
    case = synth.lf_sweep(name)
    want = lf_oracle(oracle, case)
    got = [None if p is None else p.copy() for p in case["planes"]]
    ref.ref_lf_deblock_picture(simd, *lf_args(case, got), len(case["slices"]), C.addressof(case["seq"]), 3)
    msg = lf_mismatch(oracle, case, got, want)
    assert msg is None, msg
