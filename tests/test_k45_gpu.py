"""K4 (SAO) and K5 (ALF + CC-ALF) parity on the GPU: CUDA kernels (through the C ABI) vs the pinned oracle, bit-exact."""
import ctypes as C
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth

pytestmark = pytest.mark.gpu
CASES = [(1, 256, 128, 10, 128), (2, 416, 240, 10, 64), (3, 200, 136, 8, 32), (4, 1920, 1080, 10, 128), (5, 384, 256, 12, 128),
         (6, 3840, 2160, 10, 128)]


@pytest.mark.parametrize("seed,W,H,bd,ctu", CASES)
@pytest.mark.parametrize("vb", [0, 1])
def test_sao_gpu_vs_oracle(b200, oracle, seed, W, H, bd, ctu, vb):
    rng = np.random.default_rng(seed)
    src = synth.noise_planes(rng, W, H, bd)
    sao = synth.gen_sao(rng, W, H, ctu, bd, p_on=0.7)
    sao["avail"] = np.where(rng.random(len(sao)) < 0.3, sao["avail"] & rng.integers(0, 256, size=len(sao)).astype(np.uint8), sao["avail"])
    g = abi.make_geom(W, H, bd, ctu=ctu)
    v = abi.Vb()
    if vb:
        v.numVer, v.numHor = 2, 1
        v.posX[0], v.posX[1], v.posY[0] = 8 * (W // 24), 8 * (W // 12), 8 * (H // 16)
    a = [np.zeros_like(p) for p in src]; b = [np.zeros_like(p) for p in src]
    oracle.orc_sao_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(a), sao.ctypes.data, C.addressof(v))
    vvdec_b200.check(b200.b200_sao_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(b), sao.ctypes.data, C.addressof(v)))
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c}: {np.argwhere(a[c] != b[c])[:8]}"
        assert not np.array_equal(a[c], src[c])


@pytest.mark.parametrize("seed,W,H,bd,ctu", [c for c in CASES if c[3] <= 10])
def test_alf_gpu_vs_oracle(b200, oracle, seed, W, H, bd, ctu):
    rng = np.random.default_rng(seed)
    src = synth.noise_planes(rng, W, H, bd)
    t = synth.gen_alf(rng, W, H, ctu, bd, n_aps=3)
    T = abi.make_alf_tables(t)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    a = [np.zeros_like(p) for p in src]; b = [np.zeros_like(p) for p in src]
    oracle.orc_alf_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(a), t["ctus"].ctypes.data, C.byref(T))
    vvdec_b200.check(b200.b200_alf_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(b), t["ctus"].ctypes.data, C.byref(T)))
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c}: {len(np.argwhere(a[c] != b[c]))} diffs, first {np.argwhere(a[c] != b[c])[:8]}"
        assert not np.array_equal(a[c], src[c])


@pytest.mark.parametrize("seed,W,H,bd,ctu", [(41, 416, 240, 10, 64), (42, 832, 480, 10, 128), (43, 256, 256, 8, 32)])
def test_alf_clipped_ctus_and_padded_corners(b200, oracle, seed, W, H, bd, ctu):
    """CTUs whose neighbours ALF may not read (in-loop filtering disabled across slices / tiles, AdaptiveLoopFilter.cpp:763-848): every combination of clipped sides,
    raster-slice corner padding in both forms (chroma padded with its own or with the luma margin).  The oracle's rule is pinned against the stock decoder through
    the seam (tests/test_seam_cpu.py, slices with loop filtering across them disabled)."""
    rng = np.random.default_rng(seed)
    src = synth.noise_planes(rng, W, H, bd)
    t = synth.gen_alf(rng, W, H, ctu, bd, n_aps=3, p_luma=0.9, p_chroma=0.8)
    n = len(t["ctus"])
    f = rng.integers(0, 16, size=n).astype(np.uint8) << 1                               # CLIP_TOP / BOTTOM / LEFT / RIGHT
    f = np.where(rng.random(n) < 0.3, 0, f)
    ptl = (rng.random(n) < 0.5) & ((f & (abi.ALF_CLIP_TOP | abi.ALF_CLIP_LEFT)) == 0)
    pbr = (rng.random(n) < 0.5) & ((f & (abi.ALF_CLIP_BOTTOM | abi.ALF_CLIP_RIGHT)) == 0)
    # the reference pads a corner only where that diagonal CTU exists
    ctusW = (W + ctu - 1) // ctu; ctusH = (H + ctu - 1) // ctu; idx = np.arange(n)
    ptl &= (idx % ctusW > 0) & (idx // ctusW > 0); pbr &= (idx % ctusW < ctusW - 1) & (idx // ctusW < ctusH - 1)
    f = f | (ptl * abi.ALF_PAD_TL).astype(np.uint8) | (pbr * abi.ALF_PAD_BR).astype(np.uint8)
    t["ctus"]["enable"][:, 0] |= f
    wide = (rng.random((n, 2)) < 0.5) & (f != 0)[:, None]
    t["ctus"]["ccIdx"][wide] = 0                                                        # the wide form belongs to slices without CC-ALF for that component
    t["ctus"]["enable"][:, 1:][wide] |= abi.ALF_PAD_WIDE
    assert ptl.any() and pbr.any() and (f & 30).any() and wide.any()
    T = abi.make_alf_tables(t)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    a = [np.zeros_like(p) for p in src]; b = [np.zeros_like(p) for p in src]
    oracle.orc_alf_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(a), t["ctus"].ctypes.data, C.byref(T))
    vvdec_b200.check(b200.b200_alf_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(b), t["ctus"].ctypes.data, C.byref(T)))
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c}: {len(np.argwhere(a[c] != b[c]))} diffs, first {np.argwhere(a[c] != b[c])[:8]}"


from tests.test_k45_cases_cpu import REFUSALS, refusal_variant  # noqa: E402


def _sao_call(lib, k, dst):
    return lib.b200_sao_picture(C.byref(k["g"]), abi.plane_ptrs(k["planes"]), abi.plane_ptrs(dst), k["ctus"].ctypes.data, None if k["vb"] is None else C.addressof(k["vb"]))


def _alf_call(lib, k, dst):
    T = abi.make_alf_tables(k["tables"])
    return lib.b200_alf_picture(C.byref(k["g"]), abi.plane_ptrs(k["planes"]), abi.plane_ptrs(dst), k["tables"]["ctus"].ctypes.data, C.byref(T))


def _k45_mismatch(kind, case, got, want):
    """None when every plane agrees with the oracle on the plane width and the stride padding still holds the sentinel -5; else a message naming the
    case, the plane, the first differing sample and what filters it: the ALF class / transpose of its 4x4 block, or the SAO type and EO category / band."""
    ctu = case["ctu"]
    for c, (a, b) in enumerate(zip(got, want)):
        sh = 1 if c else 0
        w = case["W"] >> sh
        if (a[:, w:] != -5).any(): return f"{case['name']}: plane {c}: the stride padding was written"
        bad = np.argwhere(a[:, :w] != b[:, :w])
        if not len(bad): continue
        y, x = (int(v) for v in bad[0])
        i = (y << sh) // ctu * ((case["W"] + ctu - 1) // ctu) + (x << sh) // ctu
        if kind == "alf":
            r = case["tables"]["ctus"][i]
            what = f"CTU {i} enable {list(r['enable'])} lumaSet {r['lumaSet']} chromaAlt {list(r['chromaAlt'])} ccIdx {list(r['ccIdx'])}"
            if c == 0:
                cs = synth.alf_class_sums(np.ascontiguousarray(case["planes"][0][:, :case["W"]]), case["bd"], ctu)
                what += f", class {cs['cls'][y // 4, x // 4]} transpose {cs['tr'][y // 4, x // 4]}"
        else:
            r = case["ctus"][i]; t = int(r["type"][c]); p = case["planes"][c].astype(np.int64)
            what = f"CTU {i} type {t} avail {r['avail']:#04x}"
            if t == 4: what += f" band {(p[y, x] >> (case['bd'] - 5)) - r['band'][c] & 31} from start {r['band'][c]}"
            elif t < 4:
                dx, dy = [(1, 0), (0, 1), (1, 1), (-1, 1)][t]
                n = [p[min(max(y + s * dy, 0), p.shape[0] - 1), min(max(x + s * dx, 0), w - 1)] for s in (-1, 1)]
                what += f" category {int(np.sign(p[y, x] - n[0]) + np.sign(p[y, x] - n[1]))}"
        return f"{case['name']}: plane {c}: {len(bad)} samples differ, first at (y={y}, x={x}): {a[y, x]} vs {b[y, x]}; {what}"
    return None


@pytest.mark.parametrize("name", list(synth.SAO_SWEEP_CASES))
def test_sao_designed_sweep(b200, oracle, name):
    """Every case of the designed SAO sweep (synth.sao_sweep): bit-exact against the oracle on the plane width, with the caller's stride padding kept."""
    case = synth.sao_sweep(name)
    want = [np.zeros_like(p) for p in case["planes"]]
    oracle.orc_sao_picture(C.byref(case["g"]), abi.plane_ptrs(case["planes"]), abi.plane_ptrs(want), case["ctus"].ctypes.data, C.addressof(case["vb"]))
    got = [np.full_like(p, -5) for p in case["planes"]]
    vvdec_b200.check(_sao_call(b200, case, got))
    msg = _k45_mismatch("sao", case, got, want)
    assert msg is None, msg


@pytest.mark.parametrize("name", list(synth.ALF_SWEEP_CASES))
def test_alf_designed_sweep(b200, oracle, name):
    """Every case of the designed ALF sweep (synth.alf_sweep): bit-exact against the oracle on the plane width, with the caller's stride padding kept."""
    case = synth.alf_sweep(name)
    T = abi.make_alf_tables(case["tables"])
    want = [np.full_like(p, -5) for p in case["planes"]]
    oracle.orc_alf_picture(C.byref(case["g"]), abi.plane_ptrs(case["planes"]), abi.plane_ptrs(want), case["tables"]["ctus"].ctypes.data, C.byref(T))
    got = [np.full_like(p, -5) for p in case["planes"]]
    vvdec_b200.check(_alf_call(b200, case, got))
    msg = _k45_mismatch("alf", case, got, want)
    assert msg is None, msg


@pytest.mark.parametrize("kind,what,bad,fixed", REFUSALS, ids=[f"{r[0]}: {r[1]}" for r in REFUSALS])
def test_k45_refusals(b200, oracle, kind, what, bad, fixed):
    """Each host rule of b200_sao_picture / b200_alf_picture, alone, makes it return B200_ERR_PARAM with an error message and dst untouched; the same call
    with the offending field fixed is accepted and equals the oracle.  The refused calls never reach the device or the oracle."""
    call = _sao_call if kind == "sao" else _alf_call
    ok = refusal_variant(kind, fixed)
    got = [np.full_like(p, -5) for p in ok["planes"]]
    assert call(b200, ok, got) == 0, (what, b200.b200_last_error())
    want = [np.full_like(p, -5) for p in ok["planes"]]
    if kind == "sao":
        oracle.orc_sao_picture(C.byref(ok["g"]), abi.plane_ptrs(ok["planes"]), abi.plane_ptrs(want), ok["ctus"].ctypes.data, C.addressof(ok["vb"]))
    else:
        T = abi.make_alf_tables(ok["tables"])
        oracle.orc_alf_picture(C.byref(ok["g"]), abi.plane_ptrs(ok["planes"]), abi.plane_ptrs(want), ok["tables"]["ctus"].ctypes.data, C.byref(T))
    nc = 3 if ok["g"].chromaFormat else 1
    for c in range(nc):
        w, h = ok["g"].width >> (c > 0), ok["g"].height >> (c > 0)
        assert np.array_equal(got[c][:h, :w], want[c][:h, :w]), (what, c)
    k = refusal_variant(kind, bad)
    dst = [np.full_like(p, -5) for p in k["planes"]]
    assert call(b200, k, dst) == -2, what
    assert f"b200_{kind}_picture".encode() in b200.b200_last_error(), what
    assert all((p == -5).all() for p in dst), what
