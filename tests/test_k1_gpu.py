"""K1 parity on the GPU: CUDA kernel (through the C ABI) vs the pinned oracle, bit-exact."""
import ctypes as C
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth

pytestmark = pytest.mark.gpu


def _run_both(b200, oracle, W, H, bd, tus, coefs, planes, mode):
    g = abi.make_geom(W, H, bd)
    a = [p.copy() for p in planes]; b = [p.copy() for p in planes]
    oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(a), tus.ctypes.data, len(tus), coefs, None, mode)
    vvdec_b200.check(b200.b200_k1_residual(C.byref(g), abi.plane_ptrs(b), tus.ctypes.data, len(tus),
                                            coefs.ctypes.data, len(coefs), None, 0, mode))
    return a, b


@pytest.mark.parametrize("seed,W,H,bd,mode", [(1, 256, 128, 10, 0), (2, 416, 240, 10, 1), (3, 256, 256, 8, 0),
                                              (4, 384, 256, 12, 1), (5, 1920, 1080, 10, 0)])
def test_k1_random_pictures(b200, oracle, seed, W, H, bd, mode):
    rng = np.random.default_rng(seed)
    cus = synth.partition(rng, W, H)
    tus, coefs = synth.gen_tus(rng, cus, bd, p_cbf=0.9, p_mts=0.25, p_lfnst=0.2, p_ts=0.1, p_bdpcm=0.1, heavy=0.05, p_intra=0.5)
    assert len(tus) > 50
    planes = synth.noise_planes(rng, W, H, bd)
    a, b = _run_both(b200, oracle, W, H, bd, tus, coefs, planes, mode)
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c} differs at {np.argwhere(a[c] != b[c])[:5]}"
    # feature coverage of this case
    if W * H >= 256 * 256:
        assert (tus["lfnst"] != 0).any() and (tus["flags"] & abi.TU_TS).any() and (tus["ict"] != 0).any()
        assert (tus["trType"] != 0).any() and (tus["flags"] & (abi.TU_BDPCM_H | abi.TU_BDPCM_V)).any()


def test_k1_every_size_dense_extreme(b200, oracle):
    """All 36 TU shapes x {DCT2, DST7, DCT8} with full corners and extreme levels (overflow wrap must match)."""
    rng = np.random.default_rng(11)
    recs, coefs, n = [], [], 0
    x = y = 0
    W = 1024
    for l2w in range(1, 7):
        for l2h in range(1, 7):
            for tr in (0, 2 | (2 << 2), 1 | (1 << 2), 2 | (1 << 2)):
                w, h = 1 << l2w, 1 << l2h
                if tr and (min(w, h) < 4 or max(w, h) > 32): continue
                limx = 16 if (tr and w == 32) else min(w, 32); limy = 16 if (tr and h == 32) else min(h, 32)
                if x + w > W: x = 0; y += 64
                lv = rng.choice(np.array([-32768, 32767, -1, 1, 0, 1234], np.int16), size=limx * limy)
                lv[-1] = 32767
                sq = (l2w + l2h) & 1
                recs.append((x, y, l2w, l2h, 0, 0, limx - 1, limy - 1, tr, 0, 0, int(rng.integers(-2, 6)), 16,
                             [64, 90][sq], n, 0, (0, 0)))
                coefs.append(lv); n += len(lv); x += w
    tus = np.array(recs, dtype=abi.TU_DTYPE); arena = np.concatenate(coefs)
    H = y + 64
    planes = [np.zeros((H, W), np.int16), np.zeros((H // 2, W // 2), np.int16), np.zeros((H // 2, W // 2), np.int16)]
    a, b = _run_both(b200, oracle, W, H, 10, tus, arena, planes, 1)
    assert np.array_equal(a[0], b[0])


def test_k1_isp_thin_partitions(b200, oracle):
    """One-sample-wide / -high luma transform units (sub-partitions of 4xN / Nx4 ISP CUs, TrQuant.cpp:466-482): a single 1-D stage with the combined shift;
    DCT-2 and the implicit DST-7 (length 16), sparse and full corners, DC-only, extreme levels.  A thin chroma block or a thin block with LFNST is refused."""
    rng = np.random.default_rng(21)
    recs, coefs, n = [], [], 0
    W, H = 512, 256
    x = y = 0
    for rep in range(6):
        for l2 in (4, 5, 6):
            for vert in (0, 1):
                for tr in ((0, 2) if l2 == 4 else (0,)):
                    w, h = (1, 1 << l2) if vert else (1 << l2, 1)
                    lim = min(1 << l2, 32)
                    m = [lim, 1, int(rng.integers(1, lim + 1))][rep % 3]
                    if x + w > W: x = 0; y += 64
                    lv = rng.choice(np.array([-32768, 32767, -1, 1, 0, 1234, -77], np.int16), size=m) if rep < 3 else rng.integers(-300, 300, size=m).astype(np.int16)
                    lv[-1] = 911
                    trType = (tr << 2) if vert else tr
                    recs.append((x, y, 0 if vert else l2, l2 if vert else 0, 0, 0, 0 if vert else m - 1, m - 1 if vert else 0, trType, 0, 0, int(rng.integers(-1, 5)), 16, [64, 90][l2 & 1], n, 0, (0, 0)))
                    coefs.append(lv); n += len(lv); x += max(w, 4)
    tus = np.array(recs, dtype=abi.TU_DTYPE); arena = np.concatenate(coefs)
    for bd, mode in ((10, 1), (8, 0), (12, 0)):
        planes = synth.noise_planes(rng, W, H, bd)
        a, b = _run_both(b200, oracle, W, H, bd, tus, arena, planes, mode)
        assert np.array_equal(a[0], b[0]), (bd, mode, np.argwhere(a[0] != b[0])[:5])
    g = abi.make_geom(W, H, 10)
    planes = synth.noise_planes(rng, W, H, 10)
    for field, val in (("comp", 1), ("lfnst", 1)):
        bad = tus[:1].copy(); bad[field] = val
        got = [p.copy() for p in planes]
        assert b200.b200_k1_residual(C.byref(g), abi.plane_ptrs(got), bad.ctypes.data, 1, arena.ctypes.data, len(arena), None, 0, 0) == -2, field
        assert b"TU record 0" in b200.b200_last_error() and all(np.array_equal(a, b) for a, b in zip(got, planes)), field


def test_k1_empty_and_errors(b200):
    g = abi.make_geom(64, 64, 10)
    planes = [np.zeros((64, 64), np.int16), np.zeros((32, 32), np.int16), np.zeros((32, 32), np.int16)]
    assert b200.b200_k1_residual(C.byref(g), abi.plane_ptrs(planes), None, 0, None, 0, None, 0, 0) == 0
    g.bitDepth = 17
    assert b200.b200_k1_residual(C.byref(g), abi.plane_ptrs(planes), None, 0, None, 0, None, 0, 0) == -2
    assert b"bit depth" in b200.b200_last_error()


@pytest.mark.parametrize("seed,W,H,bd", [(31, 416, 240, 10), (32, 256, 256, 8)])
def test_k1_explicit_scaling_lists(b200, oracle, seed, W, H, bd):
    """Explicit scaling lists (SURVEY 8a row a3, Quant.cpp:386-576 tables / :182 DeQuantScalingCore): per-position dequantisation table of the
    TU's shape, +4 right shift; TS and LFNST TUs stay flat (sps_scaling_matrix_for_lfnst_disabled)."""
    rng = np.random.default_rng(seed)
    cus = synth.partition(rng, W, H)
    sl = synth.gen_scaling_lists(rng)
    tus, coefs = synth.gen_tus(rng, cus, bd, p_cbf=0.9, p_mts=0.25, p_lfnst=0.1, p_ts=0.1, p_bdpcm=0.05, p_intra=0.5, scaling=sl)
    assert (tus["flags"] & abi.TU_SCALING).any() and not (tus["flags"] & abi.TU_SCALING).all()
    planes = synth.noise_planes(rng, W, H, bd)
    g = abi.make_geom(W, H, bd)
    a = [p.copy() for p in planes]; b = [p.copy() for p in planes]
    arena = sl["arena"]
    oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(a), tus.ctypes.data, len(tus), coefs, arena.ctypes.data, 0)
    vvdec_b200.check(b200.b200_k1_residual(C.byref(g), abi.plane_ptrs(b), tus.ctypes.data, len(tus), coefs.ctypes.data, len(coefs),
                                            arena.ctypes.data, len(arena), 0))
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c} differs at {np.argwhere(a[c] != b[c])[:5]}"
    # and the lists matter: the flat result is different
    tus2 = tus.copy(); tus2["flags"] &= ~np.uint8(abi.TU_SCALING)
    c2 = [p.copy() for p in planes]
    oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(c2), tus2.ctypes.data, len(tus2), coefs, None, 0)
    assert not np.array_equal(a[0], c2[0])


def _first_diff(case, want, got):
    """(plane, y, x, oracle sample, kernel sample, index and tags of the TUs writing it) of the first differing sample, or None."""
    for c, (a, b) in enumerate(zip(want, got)):
        if a is None or np.array_equal(a, b): continue
        y, x = (int(v) for v in np.argwhere(a != b)[0])
        t = case["tus"]
        cx, cy = t["x"].astype(int), t["y"].astype(int)
        on = ((t["comp"] == c) | ((t["ict"] != 0) & (t["comp"] == 3 - c) & (c > 0))) & (cx <= x) & (x < cx + (1 << t["log2w"].astype(int))) & (cy <= y) & (y < cy + (1 << t["log2h"].astype(int)))
        return c, y, x, int(a[y, x]), int(b[y, x]), [(int(i), case["tags"][i]) for i in np.flatnonzero(on)]
    return None


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", list(synth.K1_SWEEP_CASES))
def test_k1_designed_sweep(b200, oracle, name, mode):
    """Every case of the designed K1 sweep (synth.k1_sweep) through b200_k1_residual, bit-exact against the oracle on every plane; the stride padding keeps
    its sentinel.  A failure names the first differing sample and the TU(s) that write it."""
    case = synth.k1_sweep(name)
    g, tus, coefs, sl = case["g"], case["tus"], case["coefs"], case["scaling"]
    want, got = case["planes"], [None if p is None else p.copy() for p in case["planes"]]
    oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(want), tus.ctypes.data, len(tus), coefs, None if sl is None else sl.ctypes.data, mode)
    vvdec_b200.check(b200.b200_k1_residual(C.byref(g), abi.plane_ptrs(got), tus.ctypes.data, len(tus), coefs.ctypes.data, len(coefs),
                                            None if sl is None else sl.ctypes.data, 0 if sl is None else len(sl), mode))
    diff = _first_diff(case, want, got)
    assert diff is None, f"{name} mode {mode}: plane {diff[0]} (y {diff[1]}, x {diff[2]}): oracle {diff[3]}, kernel {diff[4]}; TU {diff[5]}"
    for c, p in enumerate(got):
        if p is not None and p.shape[1] > (case["W"] >> (c > 0)):
            assert (p[:, case["W"] >> (c > 0):] == -7).all(), f"{name}: stride padding of plane {c} written"
