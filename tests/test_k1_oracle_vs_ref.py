"""Pins oracle/k1_residual.c and the TU flattener against the reference's own functions
(oracle/_ref/libvvdec_ref.so = unmodified VVdeC + extern "C" shim). CPU only.
Pattern = vvdec_unit_test.cpp:221-303 (same call on `ref` and `opt`, random + corner inputs, exact equality)."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth
from tests.helpers import RefTuSyntax, aligned, aligned_copy

pytestmark = pytest.mark.ref


def test_simd_level(ref):
    assert ref.ref_simd_level() in (b"SCALAR", b"SSE41", b"SSE42", b"AVX", b"AVX2", b"AVX512")


@pytest.mark.parametrize("simd", [0, 1])
def test_dequant(oracle, ref, simd):
    rng = np.random.default_rng(1)
    for case in range(300):
        w = 1 << rng.integers(1, 7); h = 1 << rng.integers(1, 7)
        maxX = int(rng.integers(0, min(w, 32))); maxY = int(rng.integers(0, min(h, 32)))
        if simd:  # the SIMD dequant processes groups of 4/8 levels: the decoder always hands it w>=4 corners
            if w < 4: continue
        scale = int(rng.choice([40, 45, 51, 57, 64, 72, 80, 90, 102]))
        rs = int(rng.integers(-4, 12))
        in_bits = min(16, 32 + rs - 7)
        in_max = (1 << (in_bits - 1)) - 1
        q = rng.integers(-32768, 32768, size=(h, w)).astype(np.int16) if case % 3 == 0 else \
            (rng.laplace(0, 40, size=(h, w))).clip(-32768, 32767).astype(np.int16)
        a = np.zeros(w * h, np.int32); b = np.zeros(w * h, np.int32)
        oracle.orc_dequant(w, maxX, maxY, scale, None, q, w, a, rs, in_max, 32767)
        ref.ref_dequant(simd, w, maxX, maxY, scale, q, w, b, rs, in_max, 32767)
        assert np.array_equal(a, b), (case, w, h, maxX, maxY, scale, rs)


@pytest.mark.parametrize("simd", [0, 1])
def test_dequant_scaling_lists(oracle, ref, simd):
    """Explicit scaling lists: Quant::DeQuantScaling with a per-position table (what getDequantCoeff returns: list value, 16 = neutral)
    and the +4 right shift of LOG2_SCALING_LIST_NEUTRAL_VALUE (Quant.cpp:345)."""
    rng = np.random.default_rng(11)
    for case in range(300):
        w = 1 << rng.integers(2, 7); h = 1 << rng.integers(2, 7)
        maxX = int(rng.integers(0, min(w, 32))); maxY = int(rng.integers(0, min(h, 32)))
        scale = int(rng.choice([40, 45, 51, 57, 64, 72, 80, 90, 102]))
        rs = int(rng.integers(0, 16))
        in_bits = min(16, 32 + rs - 7)
        in_max = (1 << (in_bits - 1)) - 1
        sl = rng.integers(1, 256, size=w * h).astype(np.int32) if case % 4 else np.full(w * h, 16, np.int32)
        q = (rng.laplace(0, 40, size=(h, w))).clip(-32768, 32767).astype(np.int16)
        a = np.zeros(w * h, np.int32); b = np.zeros(w * h, np.int32)
        oracle.orc_dequant(w, maxX, maxY, scale, sl.ctypes.data, q, w, a, rs, in_max, 32767)
        ref.ref_dequant_scaling(simd, w, maxX, maxY, scale, sl, q, w, b, rs, in_max, 32767)
        assert np.array_equal(a, b), (case, w, h, maxX, maxY, scale, rs)


def test_inv_lfnst(oracle, ref):
    rng = np.random.default_rng(2)
    for case in range(400):
        size = int(rng.choice([4, 8])); zo = int(rng.choice([8, 16]))
        src = rng.integers(-32768, 32768, size=16).astype(np.int32)
        if case % 5 == 0: src[:] = rng.choice([-32768, 32767], size=16)
        a = np.zeros(48, np.int32); b = np.zeros(48, np.int32)
        st, idx = int(rng.integers(0, 4)), int(rng.integers(0, 2))
        oracle.orc_inv_lfnst(src, a, st, idx, size, zo)
        ref.ref_inv_lfnst(src.copy(), b, st, idx, size, zo)
        n = 48 if size > 4 else 16
        assert np.array_equal(a[:n], b[:n])


@pytest.mark.parametrize("simd", [0, 1])
def test_inv_1d(oracle, ref, simd):
    rng = np.random.default_rng(3)
    sizes = {abi.TR_DCT2: [2, 4, 8, 16, 32, 64], abi.TR_DCT8: [4, 8, 16, 32], abi.TR_DST7: [4, 8, 16, 32]}
    for tr, ns in sizes.items():
        for n in ns:
            for case in range(25):
                line = 1 << int(rng.integers(1, 7))
                skip_line = int(rng.choice([0, line // 2, line - min(line, 4)])) if line > 2 else 0
                if line - skip_line > 32: skip_line = line - 32
                skip2 = int(rng.choice([0, n // 2, n - 1, n - min(n, 4)]))
                if n - skip2 > 32: skip2 = n - 32
                # the decoder only produces reducedLine in {2, multiples of 4} (vvdec_unit_test.cpp:266)
                if (line - skip_line) % 4 and line - skip_line != 2: skip_line = 0
                clip = int(case & 1)
                shift = 7 if clip else 10
                lim = 32768 if (case % 4 or simd) else 1 << 20   # SIMD packs the source to 16 bit (decoder invariant; vvdec_unit_test.cpp:264 uses 16-bit inputs)
                src = aligned_copy(rng.integers(-lim, lim, size=n * line).astype(np.int32))
                if (tr == abi.TR_DCT2 and n <= 4) or simd: src[(n - skip2) * line:] = 0   # decoder invariant: rows beyond the cutoff are zero (B2/B4 butterflies and the SIMD paths rely on it)
                a = aligned(n * line, np.int32, 7); b = aligned(n * line, np.int32, 7)
                oracle.orc_inv_1d(tr, n, src, a, shift, line, skip_line, skip2, clip, -32768, 32767)
                ref.ref_inv_1d(simd, tr, n, src, b, shift, line, skip_line, skip2, clip, -32768, 32767)
                rl = line - skip_line
                assert np.array_equal(a[:rl * n], b[:rl * n]), (tr, n, line, skip_line, skip2, clip)


@pytest.mark.parametrize("simd", [0, 1])
def test_cpy_resi_clip(oracle, ref, simd):
    rng = np.random.default_rng(4)
    for case in range(100):
        w = 1 << int(rng.integers(1, 7)); h = 1 << int(rng.integers(1, 7)); stride = w + int(rng.integers(0, 9))
        src = aligned_copy(rng.integers(-(1 << 28), 1 << 28, size=w * h).astype(np.int32))
        a = aligned(h * stride, np.int16); b = aligned(h * stride, np.int16)
        oracle.orc_cpy_resi_clip(src, a, stride, w, h, -32768, 32767, 512, 10)
        ref.ref_cpy_resi_clip(simd, src, b, stride, w, h, -32768, 32767, 512, 10)
        assert np.array_equal(a, b)


def _tu_case(oracle, ref, s, levels):
    cw = s.w >> (1 if s.comp else 0); ch = s.h >> (1 if s.comp else 0)
    r0 = np.zeros(cw * ch, np.int16); r1 = np.zeros(cw * ch, np.int16)
    rec = abi.Tu(); coefs = np.zeros(cw * ch + 16, np.int16); n = C.c_int32(0)
    made = ref.ref_tu_case(C.byref(s), levels, r0, r1, C.byref(rec), coefs, C.byref(n))
    assert made == 1
    assert (1 << rec.log2w, 1 << rec.log2h) == (cw, ch)
    geom = abi.make_geom(128, 128, s.bitDepth)
    planes = [np.zeros((128, 128), np.int16), np.zeros((64, 64), np.int16), np.zeros((64, 64), np.int16)]
    recs = (abi.Tu * 1)(rec)
    oracle.orc_k1_residual(C.byref(geom), abi.plane_ptrs(planes), recs, 1, coefs, None, 1)
    coded = rec.comp
    got0 = planes[coded][:ch, :cw].reshape(-1)
    assert np.array_equal(got0, r0), ("coded comp", [(f, getattr(s, f)) for f, _ in s._fields_])
    if rec.ict:
        other = 2 if coded == 1 else 1
        assert np.array_equal(planes[other][:ch, :cw].reshape(-1), r1), "ICT plane"
    return rec


def _levels(rng, cw, ch, maxX, maxY, heavy):
    lv = np.zeros((ch, cw), np.int16)
    sub = rng.laplace(0, 6 if not heavy else 3000, size=(maxY + 1, maxX + 1)).clip(-32768, 32767).astype(np.int16)
    sub[maxY, maxX] = sub[maxY, maxX] or 1
    lv[:maxY + 1, :maxX + 1] = sub
    return lv.reshape(-1).copy()


def test_tu_level_dct2_mts_sbt(oracle, ref):
    """Whole invTransformNxN incl. flattener: DCT-2, DC-only shortcut, zero-out, explicit/implicit MTS, SBT, depQuant."""
    rng = np.random.default_rng(5)
    seen = set()
    for case in range(1500):
        s = RefTuSyntax()
        s.comp = int(rng.choice([0, 0, 1, 2]))
        s.w = 1 << int(rng.integers(2, 7)); s.h = 1 << int(rng.integers(2, 7))
        if s.comp and min(s.w, s.h) < 4: continue
        cw = s.w >> (1 if s.comp else 0); ch = s.h >> (1 if s.comp else 0)
        s.bitDepth = int(rng.choice([8, 10, 10, 12])); s.qp = int(rng.integers(-6 * (s.bitDepth - 8), 64))
        s.predMode = int(rng.integers(0, 2)); s.depQuant = int(rng.integers(0, 2))
        s.cbQpOffset = int(rng.integers(-6, 7)); s.crQpOffset = int(rng.integers(-6, 7))
        s.spsMTS = int(rng.integers(0, 2)); s.spsIntraMTS = int(rng.integers(0, 2)); s.spsInterMTS = int(rng.integers(0, 2))
        s.intraDirL = int(rng.integers(0, 67)); s.intraDirC = int(rng.integers(0, 67))
        s.maxScanPosX = int(rng.integers(0, min(cw, 32))); s.maxScanPosY = int(rng.integers(0, min(ch, 32)))
        if case % 7 == 0: s.maxScanPosX = s.maxScanPosY = 0
        if s.comp == 0 and s.spsMTS and cw <= 32 and ch <= 32:
            explicit = (s.predMode == 1 and s.spsIntraMTS) or (s.predMode == 0 and s.spsInterMTS)
            if explicit and rng.integers(0, 2):
                s.mtsIdx = int(rng.integers(2, 6))
                s.maxScanPosX = min(s.maxScanPosX, 15); s.maxScanPosY = min(s.maxScanPosY, 15)
            if s.predMode == 0 and rng.integers(0, 3) == 0 and s.mtsIdx == 0:
                s.sbtIdx = int(rng.integers(1, 5)); s.sbtPos = int(rng.integers(0, 2))
                if (s.sbtIdx in (1, 3) and cw > 32) or (s.sbtIdx in (2, 4) and ch > 32): s.sbtIdx = 0
                # sbt idx: 1 VER_HALF 2 HOR_HALF 3 VER_QUAD 4 HOR_QUAD (TypeDef.h SbtIdx); zero-out 32->16 when MTS-like
                s.maxScanPosX = min(s.maxScanPosX, 15); s.maxScanPosY = min(s.maxScanPosY, 15)
        lv = _levels(rng, cw, ch, s.maxScanPosX, s.maxScanPosY, case % 11 == 0)
        rec = _tu_case(oracle, ref, s, lv)
        seen.add(rec.trType)
    assert {0, 2 | (2 << 2), 1 | (1 << 2)} <= seen


def test_tu_level_lfnst(oracle, ref):
    rng = np.random.default_rng(6)
    seen = set()
    for case in range(800):
        s = RefTuSyntax()
        s.comp = int(rng.choice([0, 0, 1, 2])); s.predMode = 1; s.spsLFNST = 1
        s.w = 1 << int(rng.integers(2, 7)); s.h = 1 << int(rng.integers(2, 7))
        cw = s.w >> (1 if s.comp else 0); ch = s.h >> (1 if s.comp else 0)
        if min(cw, ch) < 4: continue
        s.sepTree = 1 if s.comp else 0
        s.bitDepth = 10; s.qp = int(rng.integers(10, 50)); s.depQuant = int(rng.integers(0, 2))
        s.lfnstIdx = int(rng.integers(1, 3))
        s.intraDirL = int(rng.integers(0, 67)); s.intraDirC = int(rng.choice([0, 1, 18, 50, int(rng.integers(2, 67))]))
        s.mipFlag = int(rng.integers(0, 4) == 0) if s.comp == 0 else 0
        s.spsMTS = int(rng.integers(0, 2))
        # LFNST TUs carry at most 16 (8 for 4x4/8x8) coefficients in the first CG
        s.maxScanPosX = int(rng.integers(0, 4)); s.maxScanPosY = int(rng.integers(0, 4))
        lv = _levels(rng, cw, ch, s.maxScanPosX, s.maxScanPosY, case % 9 == 0)
        rec = _tu_case(oracle, ref, s, lv)
        assert rec.lfnst & 3 == s.lfnstIdx
        seen.add(rec.lfnst >> 2)
    assert len(seen) == 7  # 4 sets x transpose; set 0 (planar/DC) is never transposed


def test_tu_level_ts_bdpcm_jccr(oracle, ref):
    rng = np.random.default_rng(7)
    icts = set()
    for case in range(900):
        s = RefTuSyntax()
        s.comp = int(rng.choice([0, 1, 2])); s.predMode = int(rng.integers(0, 2))
        s.w = 1 << int(rng.integers(2, 6)); s.h = 1 << int(rng.integers(2, 6))
        cw = s.w >> (1 if s.comp else 0); ch = s.h >> (1 if s.comp else 0)
        if min(cw, ch) < 2: continue
        s.bitDepth = int(rng.choice([8, 10])); s.qp = int(rng.integers(0, 56)); s.depQuant = int(rng.integers(0, 2))
        s.jointQpOffset = int(rng.integers(-4, 5))
        s.maxScanPosX = int(rng.integers(0, min(cw, 32))); s.maxScanPosY = int(rng.integers(0, min(ch, 32)))
        kind = case % 3
        if kind == 0:      # transform skip
            s.mtsIdx = 1
        elif kind == 1:    # BDPCM (intra, implies TS)
            s.predMode = 1; s.mtsIdx = 1
            if s.comp == 0: s.bdpcmL = int(rng.integers(1, 3))
            else: s.bdpcmC = int(rng.integers(1, 3))
        else:              # joint CbCr
            if s.comp == 0: continue
            s.jointCbCr = int(rng.integers(1, 4)); s.jointCbCrSign = int(rng.integers(0, 2))
            if rng.integers(0, 2): s.mtsIdx = 1
        lv = _levels(rng, cw, ch, s.maxScanPosX if kind != 1 else cw - 1, s.maxScanPosY if kind != 1 else ch - 1, case % 10 == 0)
        rec = _tu_case(oracle, ref, s, lv)
        if kind == 2: icts.add(rec.ict)
    assert icts == {-3, -2, -1, 1, 2, 3}


def test_tu_level_isp_thin_partitions(oracle, ref):
    """ISP groundwork: luma TUs of intra sub-partitions — 1 and 2 samples wide / high (the 1-D branches of TrQuant::xIT, :466-482) and the regular
    widths — with the implicit transform selection of ISP (getTrTypes), DC-only blocks and dependent quantisation."""
    rng = np.random.default_rng(17)
    seen = set()
    shapes = [(1, 16), (1, 32), (1, 64), (2, 8), (2, 16), (2, 32), (16, 1), (32, 1), (64, 1), (8, 2), (16, 2), (32, 2), (4, 4), (4, 16), (16, 4), (8, 8), (16, 16), (4, 32)]
    for case in range(900):
        s = RefTuSyntax()
        s.comp = 0
        s.w, s.h = shapes[case % len(shapes)]
        s.ispMode = 2 if s.w < s.h else 1 if s.h < s.w else int(rng.integers(1, 3))
        s.bitDepth = int(rng.choice([8, 10, 10, 12])); s.qp = int(rng.integers(-6 * (s.bitDepth - 8), 64))
        s.predMode = 1; s.depQuant = int(rng.integers(0, 2))
        s.spsMTS = int(rng.integers(0, 2)); s.spsIntraMTS = int(rng.integers(0, 2))
        s.intraDirL = int(rng.integers(0, 67))
        s.maxScanPosX = int(rng.integers(0, min(s.w, 32))); s.maxScanPosY = int(rng.integers(0, min(s.h, 32)))
        if case % 5 == 0: s.maxScanPosX = s.maxScanPosY = 0
        lv = _levels(rng, s.w, s.h, s.maxScanPosX, s.maxScanPosY, case % 11 == 0)
        rec = _tu_case(oracle, ref, s, lv)
        seen.add((rec.log2w, rec.log2h, rec.trType))
    assert any(k[0] == 0 for k in seen) and any(k[1] == 0 for k in seen) and len({k[2] for k in seen}) >= 3


@pytest.mark.parametrize("name", [n for n, v in synth.K1_SWEEP_CASES.items() if v[0] != "random"])
def test_k1_sweep_tus_match_the_reference(oracle, ref, name):
    """Every TU of the designed K1 sweep that has a syntax form goes through the glue's flattener and the reference's invTransformNxN
    (+ invTransformICT): the flattened record equals the sweep's field for field, and the reference's residual equals the oracle's on both planes.
    The others (level corners of part of a coefficient group, inputs past LFNST's zero-out size, 2-sample sides in luma, pairs only SBT gives, ...) are
    records only the record interface allows; the kernel is checked on them against the oracle (tests/test_k1_gpu.py)."""
    case = synth.k1_sweep(name)
    pinned = 0
    for i, (t, syn) in enumerate(zip(case["tus"], case["syntax"])):
        if syn is None: continue
        s = RefTuSyntax()
        for k, v in syn.items(): setattr(s, k, v)
        w, h = 1 << int(t["log2w"]), 1 << int(t["log2h"])
        s.maxScanPosX, s.maxScanPosY = int(t["maxX"]), int(t["maxY"])
        lv = np.zeros((h, w), np.int16)
        c = synth.k1_corner(case["tus"], case["coefs"], i)
        lv[:c.shape[0], :c.shape[1]] = c
        rec = _tu_case(oracle, ref, s, lv.reshape(-1).copy())
        got = {f: getattr(rec, f) for f in ("log2w", "log2h", "comp", "flags", "maxX", "maxY", "trType", "lfnst", "ict", "rightShift", "inBits", "scale")}
        want = {f: int(t[f]) for f in got}
        assert got == want, (name, i, case["tags"][i], {f: (got[f], want[f]) for f in got if got[f] != want[f]})
        pinned += 1
    print(f"{name}: {pinned} TUs pinned to the reference, {len(case['tus']) - pinned} record-only")
    assert pinned > len(case["tus"]) // 3
