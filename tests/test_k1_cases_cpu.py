"""The designed K1 sweep (synth.k1_sweep) on the CPU: it reaches what it is designed to reach, its saturating levels really saturate (shown with the
oracle's own dequantisation and 1-D transform), and the library accepts every record.  No GPU and no reference build needed."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth

CASES = list(synth.K1_SWEEP_CASES)


def _by_kind(kind):
    return [synth.k1_sweep(n) for n, v in synth.K1_SWEEP_CASES.items() if v[0] == kind]


def _size_class(t):
    m = max(int(t["log2w"]), int(t["log2h"]))
    return 0 if m <= 3 else 1 if m == 4 else 2 if m == 5 else 3


@pytest.mark.parametrize("name", CASES)
def test_every_sweep_record_is_legal(name):
    case = synth.k1_sweep(name)
    assert synth.k1_record_problems(case["g"], case["tus"], case["coefs"], case["scaling"]) == []
    assert len(case["tags"]) == len(case["syntax"]) == len(case["tus"])


def test_k1_record_problems_names_the_rule():
    case = synth.k1_sweep("pairs_10bit")
    bad = case["tus"].copy()
    bad[5]["lfnst"] = 3
    assert "TU record 5" in synth.k1_record_problems(case["g"], bad, case["coefs"])[0]


def test_pairs_cover_every_shape_pair_and_odd_corner():
    (case,) = _by_kind("pairs")
    tus = case["tus"]
    want = {(l2w, l2h, th | (tv << 2)) for l2w in range(1, 7) for l2h in range(1, 7) for th in synth.k1_tr_sides(1 << l2w) for tv in synth.k1_tr_sides(1 << l2h)}
    assert {(int(t["log2w"]), int(t["log2h"]), int(t["trType"])) for t in tus} == want
    mixed = {int(t["trType"]) for t in tus if (t["trType"] & 3) != (t["trType"] >> 2)}
    assert {abi.TR_DCT2 | (abi.TR_DST7 << 2), abi.TR_DST7, abi.TR_DCT8 | (abi.TR_DST7 << 2)} <= mixed
    # a 64 side beside DST-7 / DCT-8 (class 3), and the 16 x 32 zero-out of DST-7 / DCT-8 beside DCT-2 at 32
    assert any(max(t["log2w"], t["log2h"]) == 6 and t["trType"] for t in tus)
    assert any(t["log2w"] == 5 and t["log2h"] == 5 and (t["trType"] & 3) and not (t["trType"] >> 2) and t["maxX"] == 15 and t["maxY"] == 31 for t in tus)
    # DC-only corners with one DCT-2 side and one DST-7 / DCT-8 side (no DC shortcut)
    assert any(t["maxX"] == 0 and t["maxY"] == 0 and ((t["trType"] & 3) == 0) != ((t["trType"] >> 2) == 0) for t in tus)
    for cls in range(4):
        lim = (8, 16, 32, 32)[cls]
        sub = [t for t in tus if _size_class(t) == cls]
        for v in (o for o in synth.K1_ODD if o <= lim):
            assert any(int(t["maxX"]) + 1 == v for t in sub) and any(int(t["maxY"]) + 1 == v for t in sub), (cls, v)
    # most TUs of every size class are dense (a sparse TU then inherits non-zero shared memory)
    for cls in range(4):
        sub = [t for t in tus if _size_class(t) == cls]
        dense = [t for t in sub if (int(t["maxX"]) + 1) * (int(t["maxY"]) + 1) >= 4]
        assert len(dense) * 2 > len(sub), cls


def test_lfnst_covers_every_set_index_transpose_form_and_input():
    (case,) = _by_kind("lfnst")
    seen, full = set(), set()
    for i, t in enumerate(case["tus"]):
        w, h = 1 << int(t["log2w"]), 1 << int(t["log2h"])
        key = (int(t["lfnst"]) >> 2 & 3, int(t["lfnst"]) & 3, int(t["lfnst"]) >> 4, synth.k1_lfnst_form(w, h), t["comp"] > 0)
        c = synth.k1_corner(case["tus"], case["coefs"], i)
        nz = [synth.K1_SCAN.index((int(y), int(x))) for y, x in np.argwhere(c)]
        if len(nz) == 1: seen.add(key + (nz[0],))
        if len(nz) == 16 and (np.abs(c.astype(int)) >= 32767).all(): full.add(key)
    combos = [(s, i, tp) for (s, tp) in synth.K1_LFNST_MODES for i in (1, 2)]
    assert len(combos) == 14
    for form in synth.K1_LFNST_SHAPES:
        for s, i, tp in combos:
            assert all(any((s, i, tp, form, ch, p) in seen for ch in (False, True)) for p in range(16)), (s, i, tp, form)
            assert any((s, i, tp, form, ch) in full for ch in (False, True)), (s, i, tp, form)
    # luma and dual-tree chroma, 64 x 64 in class 3
    assert {k[4] for k in seen} == {False, True}
    assert any(t["log2w"] == 6 and t["log2h"] == 6 for t in case["tus"])


def test_dequant_covers_qps_scales_shifts_and_scaling_extremes():
    cases = _by_kind("dequant")
    assert sorted(c["bd"] for c in cases) == [8, 9, 10, 12]
    for c in cases:
        tus, bd = c["tus"], c["bd"]
        assert {int(s) for s in tus["scale"]} == {s for row in synth.TU_INV_SCALES for s in row}
        # the most negative shift the decoder can produce (2x2 chroma at QP 63, no dependent quantisation) and positive shifts
        most = synth.tu_dequant(63 + 6 * (bd - 8), bd, 1, 1)[0]
        assert int(min(t["rightShift"] for t, tag in zip(tus, c["tags"]) if tag.startswith("dequant QP"))) == most and int(tus["rightShift"].max()) > 0
        syn = [s for s in c["syntax"] if s]
        assert {s["qp"] for s in syn} == set(range(-6 * (bd - 8), 64)) and {s["depQuant"] for s in syn} == {0, 1}
        sl = tus[(tus["flags"] & abi.TU_SCALING) != 0]
        assert len(sl) and set(c["scaling"].tolist()) == {1, 255}


def test_dequant_clips_and_wraps_bind(oracle):
    """The inMax clip changes a dequantised coefficient (orc_dequant with the record's inMax differs from the same call with inMax 32767), and the left
    shift wraps in 32 bits (orc_dequant differs from the exact product saturated to 16 bits)."""
    clip = wrap = 0
    for c in _by_kind("dequant"):
        for i, t in enumerate(c["tus"]):
            lv = np.ascontiguousarray(synth.k1_corner(c["tus"], c["coefs"], i))
            h, w = lv.shape
            sl = c["scaling"][t["slOff"]:].ctypes.data if t["flags"] & abi.TU_SCALING else None
            a, b = np.zeros(w * h, np.int32), np.zeros(w * h, np.int32)
            inmax = (1 << (int(t["inBits"]) - 1)) - 1
            oracle.orc_dequant(w, w - 1, h - 1, int(t["scale"]), sl, lv, w, a, int(t["rightShift"]), inmax, 32767)
            oracle.orc_dequant(w, w - 1, h - 1, int(t["scale"]), sl, lv, w, b, int(t["rightShift"]), 32767, 32767)
            clip += int((a != b).any())
            if t["rightShift"] < 0:
                f = c["scaling"][t["slOff"]:t["slOff"] + w * h].astype(object) if t["flags"] & abi.TU_SCALING else 1
                exact = np.clip(lv.reshape(-1).astype(object).clip(-inmax - 1, inmax) * f * int(t["scale"]) * 2 ** -int(t["rightShift"]), -32768, 32767)
                wrap += int((a.astype(object) != exact).any())
    assert clip >= 8 and wrap >= 8, (clip, wrap)


def test_stage1_sums_leave_int16(oracle):
    """Saturating levels make the stage-1 (vertical) sums leave int16 before clip16, in every size class and for every vertical transform: orc_inv_1d
    without its clip, on the coefficients orc_dequant makes."""
    (case,) = _by_kind("pairs")
    seen = set()
    for i, t in enumerate(case["tus"]):
        if "saturating" not in case["tags"][i]: continue
        w, h = 1 << int(t["log2w"]), 1 << int(t["log2h"])
        lv = np.ascontiguousarray(synth.k1_corner(case["tus"], case["coefs"], i))
        dq = np.zeros(w * h, np.int32)
        oracle.orc_dequant(w, int(t["maxX"]), int(t["maxY"]), int(t["scale"]), None, lv, lv.shape[1], dq, int(t["rightShift"]), (1 << (int(t["inBits"]) - 1)) - 1, 32767)
        out = np.zeros(w * h, np.int32)
        oracle.orc_inv_1d(int(t["trType"]) >> 2, h, dq, out, 7, w, 0, 0, 0, -32768, 32767)
        s1 = (out.astype(np.int64) + 64) >> 7
        if (np.abs(s1) > 32767).any(): seen.add((_size_class(t), int(t["trType"]) >> 2))
    assert {(c, tr) for c in range(4) for tr in (0, 1, 2) if c < 3 or tr == 0} <= seen | {(0, 1), (0, 2)} and (0, 0) in seen, seen


def test_bdpcm_running_sums_saturate():
    for case in _by_kind("ts_bdpcm"):
        sat = set()
        for i, t in enumerate(case["tus"]):
            f = int(t["flags"])
            if not f & (abi.TU_BDPCM_H | abi.TU_BDPCM_V): continue
            lv = synth.k1_corner(case["tus"], case["coefs"], i).astype(np.int64)
            s = np.cumsum(lv, axis=1 if f & abi.TU_BDPCM_H else 0)
            if (s > 32767).any() and (s < -32768).any(): sat.add((f & (abi.TU_BDPCM_H | abi.TU_BDPCM_V), t["comp"] > 0))
        assert sat == {(abi.TU_BDPCM_H, False), (abi.TU_BDPCM_V, False), (abi.TU_BDPCM_H, True), (abi.TU_BDPCM_V, True)}
        ts = case["tus"][(case["tus"]["flags"] & abi.TU_TS) != 0]
        assert {(int(t["log2w"]), int(t["log2h"])) for t in ts} >= {(a, b) for a in range(2, 6) for b in range(2, 6)} | {(a, b) for a in range(1, 5) for b in range(1, 5)}


def test_jccr_covers_every_ict_on_both_planes_with_odd_negative_residuals():
    for case in _by_kind("jccr"):
        tus = case["tus"]
        assert {(int(t["ict"]), int(t["comp"])) for t in tus} == {(m, c) for m in (1, -1, 2, -2, 3, -3) for c in (1, 2)}
        vals = set()
        for i, t in enumerate(tus):
            if t["flags"] & abi.TU_TS: vals |= set(synth.k1_corner(tus, case["coefs"], i).reshape(-1).tolist())
        assert {-32768, -1, 1, -3, -5, 32767} <= vals
        pmax = (1 << case["bd"]) - 1
        assert all({0, pmax} == set(np.unique(p[:, :case["W"] >> 1]).tolist()) for p in case["planes"][1:])


def test_geometry_cases():
    k = {n: synth.k1_sweep(n) for n, v in synth.K1_SWEEP_CASES.items() if v[0] == "random"}
    assert k["geometry_400"]["g"].chromaFormat == 0 and (k["geometry_400"]["tus"]["comp"] == 0).all()
    assert {c["bd"] for c in k.values()} >= {9, 10, 12} and any(s % 2 for c in k.values() if c["strides"] for s in c["strides"])
    c = k["uhd_3840x2160"]
    assert (c["W"], c["H"]) == (3840, 2160)
    for c in k.values():
        t = c["tus"]
        right = t["x"].astype(int) + (1 << t["log2w"].astype(int)) == np.where(t["comp"] > 0, c["W"] >> 1, c["W"])
        bottom = t["y"].astype(int) + (1 << t["log2h"].astype(int)) == np.where(t["comp"] > 0, c["H"] >> 1, c["H"])
        assert right.any() and bottom.any(), c["name"]
