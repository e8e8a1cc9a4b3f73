"""K6 intra prediction on the device (b200_intra_predict / b200_intra_reconstruct) against the oracle, which tests/test_intra_oracle_vs_ref.py
pins to the real IntraPrediction, and against the golden all-intra picture produced by the reference itself.  Whole pictures are predicted as one
list: every block reads what the blocks before it produced, so a single wrong sample (or a missed dependency) spreads over the picture.

K6 has two kernels, chosen by list density: one CTA per block (v1, sparse lists: the intra blocks of B pictures) and one CTA per CTU (v2, dense lists:
I pictures).  Every list here runs under each setting of tests.helpers.INTRA_KERNELS (auto, v1, v1 in list order, v2) against one oracle result."""
import ctypes as C
import functools
import os
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth
from tests import helpers
from tests.helpers import INTRA_KERNELS, intra_run, assert_planes_equal

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "k6_intra_picture.npz")
_oracle = functools.lru_cache(maxsize=None)(helpers.load_oracle)


def _reconstruct(g, planes, resi, recs):
    want = [None if p is None else p.copy() for p in planes]
    if resi is None: _oracle().orc_intra_predict(C.byref(g), abi.plane_ptrs(want), recs.ctypes.data, len(recs))
    else: _oracle().orc_intra_reconstruct(C.byref(g), abi.plane_ptrs(want), abi.plane_ptrs(resi), recs.ctypes.data, len(recs))
    return want


@functools.lru_cache(maxsize=None)
def _picture_case(W, H, bd, ctu, min_size, p_resi, seed):
    rng = np.random.default_rng(seed)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    layout = synth.gen_intra_layout(rng, W, H, ctu, min_size=min_size)
    recs = synth.gen_intra_records(rng, layout, W, H, p_resi=p_resi, p_lm=0.25, colloc=seed & 1, ctu=ctu)
    planes = synth.noise_planes(rng, W, H, bd)
    resi = [rng.integers(-40, 41, size=p.shape).astype(np.int16) for p in planes]
    return g, planes, resi, recs, _reconstruct(g, planes, resi, recs)


def _every_kernel(b200, g, planes, recs, want, resi=None, kernels=INTRA_KERNELS):
    """Runs the list under each K6 setting against one oracle result; a failure names every setting that differs, each with its first differing samples."""
    bad = []
    for kernel in kernels:
        try: assert_planes_equal(intra_run(b200, kernel, g, planes, recs, resi), want, kernel)
        except AssertionError as e: bad.append(str(e))
    assert not bad, bad


@pytest.mark.parametrize("W,H,bd,ctu,min_size,p_resi,seed", [(256, 128, 10, 128, 8, 0.0, 1), (192, 128, 10, 64, 4, 0.5, 2), (416, 240, 8, 128, 8, 0.5, 3),
                                                             (832, 480, 10, 128, 4, 0.3, 4), (1920, 1080, 10, 128, 8, 0.5, 5), (256, 256, 12, 64, 4, 1.0, 6)])
def test_intra_picture_vs_oracle(b200, W, H, bd, ctu, min_size, p_resi, seed):
    g, planes, resi, recs, want = _picture_case(W, H, bd, ctu, min_size, p_resi, seed)
    _every_kernel(b200, g, planes, recs, want, resi)
    assert len(np.unique(recs["mode"])) > 40 and (recs["multiRefIdx"] > 0).any() and (recs["mode"] == 67).any() and (recs["mode"] == abi.INTRA_MIP).any()
    assert all((recs["mode"] == m).any() for m in (abi.INTRA_LM, abi.INTRA_MDLM_L, abi.INTRA_MDLM_T))


@functools.lru_cache(maxsize=None)
def _isp_case(W, H, bd, ctu, min_size, seed):
    rng = np.random.default_rng(seed)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    layout = synth.gen_intra_layout(rng, W, H, ctu, min_size=min_size)
    recs = synth.gen_intra_records(rng, layout, W, H, p_resi=0.5, p_lm=0.2, p_isp=0.4, ctu=ctu)
    planes = synth.noise_planes(rng, W, H, bd)
    resi = [rng.integers(-40, 41, size=p.shape).astype(np.int16) for p in planes]
    return g, planes, resi, recs, _reconstruct(g, planes, resi, recs)


@pytest.mark.parametrize("W,H,bd,ctu,min_size,seed", [(256, 128, 10, 128, 4, 11), (416, 240, 8, 64, 4, 12), (832, 480, 10, 128, 8, 13), (1920, 1080, 10, 128, 4, 14)])
def test_intra_sub_partitions_vs_oracle(b200, W, H, bd, ctu, min_size, seed):
    """ISP CUs among regular ones (one record per prediction region, thin regions, per-TU residual masks).  These lists are dense: under auto they run
    the CTU-resident kernel."""
    g, planes, resi, recs, want = _isp_case(W, H, bd, ctu, min_size, seed)
    isp = recs[(recs["flags"] & abi.INTRA_ISP) != 0]
    assert len(isp) > 20 and ((isp["mip"] & 3) == 2).any()
    if min_size == 4: assert (isp["log2h"] == 0).any() and (isp["ciip"] > 1).any() and (((isp["mip"] >> 4) & 3) == 0).any()      # 1-high regions, several TUs in a region, 4-wide CUs
    _every_kernel(b200, g, planes, recs, want, resi)
    # a region whose predecessor is missing is refused (the host checks the records before either kernel runs)
    k = int(np.flatnonzero(((recs["flags"] & abi.INTRA_ISP) != 0) & (((recs["mip"] >> 2) & 3) == 1))[0])
    broken = np.delete(recs, k - 1)
    for kernel in ("v1", "v2"):
        got = [p.copy() for p in planes]
        with helpers.intra_kernel(kernel):
            assert b200.b200_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), broken.ctypes.data, len(broken)) == -2 and b"ISP" in b200.b200_last_error()


@functools.lru_cache(maxsize=None)
def _golden():
    z = np.load(GOLD)
    W, H, bd, ctu = [int(v) for v in z["geom"]]
    g = abi.make_geom(W, H, bd, ctu=ctu)
    src = [np.ascontiguousarray(z[f"src{c}"]) for c in range(3)]; resi = [np.ascontiguousarray(z[f"resi{c}"]) for c in range(3)]
    recs = np.ascontiguousarray(z["recs"])
    return g, src, resi, recs, [np.ascontiguousarray(z[f"out{c}"]) for c in range(3)], _reconstruct(g, src, None, recs)


def test_intra_predict_only_and_golden(b200):
    g, src, resi, recs, out, want_pred = _golden()
    _every_kernel(b200, g, src, recs, out, resi)
    # prediction only (no residual planes): the flag is ignored
    _every_kernel(b200, g, src, recs, want_pred)


@functools.lru_cache(maxsize=None)
def _sweep(reconstruct):
    W, H, recs = synth.intra_sweep()
    rng = np.random.default_rng(40)
    g = abi.make_geom(W, H, 10)
    planes = [rng.integers(0, 1 << 10, size=(h, w)).astype(np.int16) for (w, h) in ((W, H), (W // 2, H // 2), (W // 2, H // 2))]
    resi = [rng.integers(-64, 65, size=p.shape).astype(np.int16) for p in planes] if reconstruct else None
    return g, planes, resi, recs, _reconstruct(g, planes, resi, recs)


@pytest.mark.parametrize("kernel", INTRA_KERNELS)
@pytest.mark.parametrize("reconstruct", [False, True], ids=["predict", "reconstruct"])
def test_intra_designed_sweep(b200, kernel, reconstruct):
    """Every (component, shape, mode) combination K6 takes, MRL, BDPCM and every MIP mode, each with a full, a partial and no neighbourhood, on noise
    (tests/test_k6_cases_cpu.py checks that the list covers all of it and that no block reads another)."""
    g, planes, resi, recs, want = _sweep(reconstruct)
    assert_planes_equal(intra_run(b200, kernel, g, planes, recs, resi), want, kernel)


@functools.lru_cache(maxsize=None)
def _geometry_case(name):
    g, planes, resi, recs = helpers.intra_case(**helpers.INTRA_CASES[name])
    return g, planes, resi, recs, _reconstruct(g, planes, resi, recs)


@pytest.mark.parametrize("kernel", INTRA_KERNELS)
@pytest.mark.parametrize("name", list(helpers.INTRA_CASES))
def test_intra_geometry_vs_oracle(b200, name, kernel):
    """CTU 32, partial CTUs, strides that are not a multiple of 8 samples (4-byte tile staging) or odd (v1 only), 4:0:0, 8 and 12 bit, CTUs with more
    records than the CTU-resident kernel stages (1024), and a sparse list of intra and CIIP blocks (the B-picture regime)."""
    g, planes, resi, recs, want = _geometry_case(name)
    assert_planes_equal(intra_run(b200, kernel, g, planes, recs, resi), want, (name, kernel))


def test_intra_argument_checks(b200):
    g = abi.make_geom(256, 128, 10)
    planes = [np.zeros((128, 256), np.int16), np.zeros((64, 128), np.int16), np.zeros((64, 128), np.int16)]
    r = np.zeros(1, abi.INTRA_TU_DTYPE)
    r["x"], r["y"], r["log2w"], r["log2h"], r["mode"] = 248, 0, 4, 4, 0
    assert b200.b200_intra_predict(C.byref(g), abi.plane_ptrs(planes), r.ctypes.data, 1) == -2 and b"geometry" in b200.b200_last_error()
    r["x"], r["numAbove"] = 0, 3
    assert b200.b200_intra_predict(C.byref(g), abi.plane_ptrs(planes), r.ctypes.data, 1) == -2 and b"availability" in b200.b200_last_error()


@pytest.mark.parametrize("kernel", INTRA_KERNELS)
def test_intra_refuses_block_across_ctus(b200, kernel):
    """A block that is not inside one CTU (chroma: half the CTU size) is refused, and the next list runs."""
    g, planes, resi, recs, want = _picture_case(192, 128, 10, 64, 4, 0.5, 2)
    for comp, x, y, l2w, l2h in ((0, 56, 0, 4, 3), (0, 0, 60, 2, 3), (1, 24, 0, 4, 2), (2, 0, 28, 2, 3)):
        bad = recs.copy()
        i = int(np.flatnonzero(bad["comp"] == comp)[0])
        bad[i]["x"], bad[i]["y"], bad[i]["log2w"], bad[i]["log2h"], bad[i]["numAbove"], bad[i]["numLeft"], bad[i]["flags"] = x, y, l2w, l2h, 0, 0, 0
        bad[i]["mode"], bad[i]["multiRefIdx"] = 0, 0
        got = [p.copy() for p in planes]
        with helpers.intra_kernel(kernel):
            assert b200.b200_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), bad.ctypes.data, len(bad)) == -2
        assert b"not inside one CTU" in b200.b200_last_error(), (comp, x, y)
    assert_planes_equal(intra_run(b200, kernel, g, planes, recs, resi), want, kernel)


@pytest.mark.parametrize("kernel", INTRA_KERNELS)
def test_intra_ctu_block_limit(b200, kernel):
    """Overlapping records can put more blocks into one CTU than the CTU-resident kernel has done bytes for (3072).  That kernel refuses such a list
    before it stages anything; the one-CTA-per-block kernel reconstructs it (the repeated block writes the same samples every time)."""
    g, planes, resi, recs, want = _picture_case(256, 128, 10, 128, 8, 0.0, 1)
    r = np.zeros(1, abi.INTRA_TU_DTYPE)
    r["x"], r["y"], r["log2w"], r["log2h"], r["mode"], r["numAbove"], r["numLeft"], r["flags"] = 8, 8, 2, 2, 50, 2, 2, abi.INTRA_AVAIL_TL | abi.INTRA_ADD_RESI
    many = np.ascontiguousarray(np.repeat(r, 3100))
    assert helpers.intra_dense(g, len(many))
    got = [p.copy() for p in planes]
    with helpers.intra_kernel(kernel):
        rc = b200.b200_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), many.ctypes.data, len(many))
    if kernel in ("auto", "v2"):
        assert rc == -2 and b"more than 3072" in b200.b200_last_error()
    else:
        assert rc == 0, b200.b200_last_error()
        assert_planes_equal(got, _reconstruct(g, planes, resi, many), kernel)
    assert_planes_equal(intra_run(b200, kernel, g, planes, recs, resi), want, kernel)
