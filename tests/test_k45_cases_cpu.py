"""The designed K4 / K5 sweep (synth.sao_sweep, synth.alf_sweep) on the CPU: the classification restatement (synth.alf_class_sums) equals the oracle's
on every block, the sweep reaches every ALF class x transpose, activity and comparison side, every SAO category x class, every avail mask with every
class, every band start with samples in and just outside its four bands, and the clips of both filters.  Also: b200_sao_picture / b200_alf_picture,
asked through synth.k45_record_problems (their checks all run on the host), accept the generated, golden and sweep records and refuse each row of
the refusal table (tests/test_k45_gpu.py runs the accepted calls)."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth
from tests.test_golden_cpu import k4_inputs, k5_inputs

SAO_CASES = list(synth.SAO_SWEEP_CASES)
ALF_CASES = list(synth.ALF_SWEEP_CASES)


def _sgn(v):
    return np.sign(v).astype(np.int64)


@pytest.mark.parametrize("name", ALF_CASES)
def test_class_sums_equal_oracle(oracle, name):
    """alf_class_sums gives every 4x4 block of the case the class and transpose orc_alf_classify gives it (32x32 blocks on the padded picture)."""
    case = synth.alf_sweep(name)
    W, H, bd, ctu = case["W"], case["H"], case["bd"], case["ctu"]
    plane = np.ascontiguousarray(case["planes"][0][:, :W])
    cs = synth.alf_class_sums(plane, bd, ctu)
    padded = np.pad(plane, 8, mode="edge")
    org = padded.ctypes.data + 2 * (8 * padded.shape[1] + 8)
    cls = np.zeros(64, np.uint16)
    for by in range(0, H, 32):
        for bx in range(0, W, 32):
            bw, bh = min(32, W - bx), min(32, H - by)
            oracle.orc_alf_classify(cls.ctypes.data, org, padded.shape[1], bx, by, bw, bh, bd + 4, ctu, ctu - 4)
            got = cls.reshape(8, 8)[:bh // 4, :bw // 4]
            want_c, want_t = cs["cls"][by // 4:(by + bh) // 4, bx // 4:(bx + bw) // 4], cs["tr"][by // 4:(by + bh) // 4, bx // 4:(bx + bw) // 4]
            assert np.array_equal(got & 0xff, want_c) and np.array_equal(got >> 8, want_t), (name, bx, by)


def test_alf_sweep_covers_classes_comparisons_and_tables():
    """Every class x transpose, every activity 0..15, each of sV > sH, sD0 > sD1, d1*hv0 > hv1*d0, hvd1 > 2*hvd0 and 2*hvd1 > 9*hvd0 on both sides and at
    equality with nonzero sides, virtual-boundary rows with activity 0 and above; the tables hold -128, 127, +128 (a set with it on every tap, one with it
    on a single tap per class) and 0; every CC-ALF value -64..64, ccIdx 1..4 and chromaAlt 0..7 on enabled CTUs, every lumaSet 0..23, CC-ALF with chroma
    ALF off, unfiltered CTUs beside filtered ones; every CLIP combination, PAD_TL, PAD_BR and PAD_WIDE; 8 / 9 / 10 bit, CTU 32 / 64 / 128, 4:0:0,
    padded strides, chroma widths of 4 mod 8, last CTU rows of ctu - 8 and of ctu, and a 3840x2160 picture."""
    keys, cc, sets, alts, ccidx, clips, bds, ctus, flags = set(), set(), set(), set(), set(), set(), set(), set(), set()
    cc_without_chroma = unfiltered = wide = False
    geo = set()
    for name in ALF_CASES:
        case = synth.alf_sweep(name)
        t, a = case["tables"], case["tables"]["ctus"]
        keys |= synth.alf_class_keys(synth.alf_class_sums(np.ascontiguousarray(case["planes"][0][:, :case["W"]]), case["bd"], case["ctu"]))
        for c in range(2): cc |= set(t["cc"][c].ravel().tolist())
        on = a["enable"][:, 0] & 1 == 1
        sets |= set(a["lumaSet"][on].tolist()); unfiltered |= bool(on.any() and (~on).any())
        for c in range(2):
            con = a["enable"][:, 1 + c] & 1 == 1
            alts |= set(a["chromaAlt"][con, c].tolist()); ccidx |= set(a["ccIdx"][:, c].tolist())
            cc_without_chroma |= bool(((a["ccIdx"][:, c] > 0) & ~con).any())
            wide |= bool((a["enable"][:, 1 + c] & 2).any())
        flags |= set((a["enable"][:, 0] & 0x7e).tolist())
        clips.add(tuple(np.unique(t["lumaClip"][16:]).tolist()))
        bds.add(case["bd"]); ctus.add(case["ctu"])
        if not case["chroma"]: geo.add("400")
        if case["strides"]: geo.add("strides")
        if case["chroma"] and (case["W"] // 2) % 8 == 4: geo.add("chroma 4 mod 8")
        if case["H"] % case["ctu"] == case["ctu"] - 8: geo.add("last ctu-8")
        if case["H"] % case["ctu"] == 0 and case["H"] > case["ctu"]: geo.add("last full")
        if (case["W"], case["H"]) == (3840, 2160): geo.add("4k")
    want = {("ct", c, t) for c in range(25) for t in range(4)} | {("act", a) for a in range(16)} | {("cmp", k, s) for k in range(5) for s in (-1, 0, 1)}
    assert want | {("vb", False), ("vb", True)} <= keys, sorted(want - keys)
    t = synth.alf_sweep("coeffs_10bit_ctu32_last24")["tables"]
    L = t["lumaCoeff"][16:, 0, :, :12]
    assert {-128, 127, 128, 0} <= set(L.ravel().tolist())
    assert (L == 128).all(axis=(1, 2)).any() and any(((s == 128).sum(axis=1) == 1).all() for s in L)
    assert {-128, 128} <= set(t["chromaCoeff"][:, :6].ravel().tolist()) and len(np.unique(t["chromaClip"])) == 4
    assert set(range(-64, 65)) <= cc, sorted(set(range(-64, 65)) - cc)
    assert sets == set(range(24)) and alts == set(range(8)) and ccidx >= {1, 2, 3, 4}
    assert all(len(c) == 4 for c in clips)
    assert cc_without_chroma and unfiltered and wide
    assert {f & 0x1e for f in flags} == set(range(0, 32, 2)) and any(f & 32 for f in flags) and any(f & 64 for f in flags)
    assert bds == {8, 9, 10} and ctus == {32, 64, 128}
    assert geo == {"400", "strides", "chroma 4 mod 8", "last ctu-8", "last full", "4k"}, geo


def _sao_ctu_stats(case):
    """Per CTU and component: ('eo', class, category) / ('bo', start, band - start) for every sample whose neighbours lie inside the CTU, and whether
    the unclipped result leaves [0, pmax] below / above."""
    g, bd, ctu = case["g"], case["bd"], case["ctu"]
    pmax = (1 << bd) - 1
    seen, clip = set(), set()
    ctusW = (case["W"] + ctu - 1) // ctu
    for i, r in enumerate(case["ctus"]):
        cx, cy = i % ctusW, i // ctusW
        for c in range(3 if case["chroma"] else 1):
            t = int(r["type"][c])
            if t == 255: continue
            sh = 1 if c else 0
            x0, y0, s = (cx * ctu) >> sh, (cy * ctu) >> sh, ctu >> sh
            blk = case["planes"][c][y0:y0 + s, x0:x0 + s].astype(np.int64)
            blk = blk[:, :min(s, (case["W"] >> sh) - x0)]
            if t == 4:
                rel = ((blk >> (bd - 5)) - int(r["band"][c])) & 31
                seen |= {("bo", int(r["band"][c]), int(v)) for v in np.unique(rel)}
                off = np.zeros(32, np.int64); off[:4] = r["offset"][c][:4]
                v = blk + off[rel]
            else:
                dx, dy = [(1, 0), (0, 1), (1, 1), (-1, 1)][t]
                ctr = blk[1:-1, 1:-1]
                h, w = blk.shape
                n0 = blk[1 - dy:h - 1 - dy, 1 - dx:w - 1 - dx]; n1 = blk[1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx]
                e = _sgn(ctr - n0) + _sgn(ctr - n1)
                seen |= {("eo", t, int(k)) for k in np.unique(e)}
                v = ctr + np.array(r["offset"][c], np.int64)[e + 2]
            if (v < 0).any(): clip.add("low")
            if (v > pmax).any(): clip.add("high")
    return seen, clip


def test_sao_sweep_covers_categories_bands_masks_and_clips():
    """Every EO class x category -2..2 (plateaus included) and every BO start 0..31 with samples in each of its four bands and in the bands just before
    and after, at 8, 9, 10 and 12 bit with the largest legal offsets; results past 0 and past pmax; every avail mask with every luma class on interior
    CTUs (and every mask on chroma EO); 0..3 vertical and horizontal virtual boundaries, at 8, at W - 8, on CTU edges and at 8 mod 16; CTU 32 / 64 / 128,
    partial CTUs, 4:0:0, padded strides and a 3840x2160 picture."""
    seen, clip, bo_bd, vers, hors, vb_forms, ctus, geo = set(), set(), set(), set(), set(), set(), set(), set()
    for name in SAO_CASES:
        case = synth.sao_sweep(name)
        s, cl = _sao_ctu_stats(case)
        seen |= s; clip |= cl
        M = synth.sao_max_offset(case["bd"])
        if case["kind"] == "bo": bo_bd.add((case["bd"], int(np.abs(case["ctus"]["offset"][:, :, :4]).max()) == M))
        vb = case["vb"]
        vers.add(vb.numVer); hors.add(vb.numHor)
        for k in range(vb.numVer):
            x = vb.posX[k]
            vb_forms |= {f for f, ok in (("at 8", x == 8), ("at W-8", x == case["W"] - 8), ("ctu edge", x % case["ctu"] == 0), ("8 mod 16", x % 16 == 8)) if ok}
        ctus.add(case["ctu"])
        if not case["chroma"]: geo.add("400")
        if case["strides"]: geo.add("strides")
        if case["W"] % case["ctu"]: geo.add("partial")
        if (case["W"], case["H"]) == (3840, 2160): geo.add("4k")
    assert {("eo", t, e) for t in range(4) for e in range(-2, 3)} <= seen
    assert {("bo", b, k) for b in range(32) for k in (0, 1, 2, 3, 4, 31)} <= seen
    assert bo_bd == {(8, True), (9, True), (10, True), (12, True)} and clip == {"low", "high"}
    assert vers == hors == {0, 1, 2, 3} and vb_forms == {"at 8", "at W-8", "ctu edge", "8 mod 16"}
    assert ctus == {32, 64, 128} and geo == {"400", "strides", "partial", "4k"}
    m = synth.sao_sweep("avail_masks_ctu32")
    W = m["W"]; ctusW = (W + 31) // 32; ctusH = (m["H"] + 31) // 32
    inner = [i for i in range(len(m["ctus"])) if 0 < i % ctusW < ctusW - 1 and 0 < i // ctusW < ctusH - 1]
    assert {(int(m["ctus"]["avail"][i]), int(m["ctus"]["type"][i, 0])) for i in inner} == {(a, t) for a in range(256) for t in range(4)}
    assert {int(m["ctus"]["avail"][i]) for i in inner if m["ctus"]["type"][i, 1] < 4} == set(range(256))


def test_rule_accepts_generated_golden_and_sweep_records():
    for seed, W, H, ctu, bd in [(1, 256, 128, 128, 10), (2, 416, 240, 64, 10), (3, 200, 136, 32, 8), (5, 384, 256, 128, 12)]:
        rng = np.random.default_rng(seed)
        g = abi.make_geom(W, H, bd, ctu=ctu)
        assert synth.k45_record_problems("sao", g, synth.gen_sao(rng, W, H, ctu, bd)) == [], seed
        if bd <= 10:
            t = synth.gen_alf(rng, W, H, ctu, bd, n_aps=3)
            assert synth.k45_record_problems("alf", g, t["ctus"], t) == [], seed
    z, g, src, sao, v = k4_inputs()
    assert synth.k45_record_problems("sao", g, sao, vb=v) == []
    z, g, src, t, T = k5_inputs()
    assert synth.k45_record_problems("alf", g, t["ctus"], t) == []
    for name in SAO_CASES:
        case = synth.sao_sweep(name)
        assert synth.k45_record_problems("sao", case["g"], case["ctus"], vb=case["vb"]) == [], name
    for name in ALF_CASES:
        case = synth.alf_sweep(name)
        assert synth.k45_record_problems("alf", case["g"], case["tables"]["ctus"], case["tables"]) == [], name


# ---- refusals: a small legal base call per filter and one edit per rule (the GPU file runs each through b200_sao_picture / b200_alf_picture)
def refusal_base(kind):
    """64 x 64, 10 bit, 4:2:0, CTU 32 (2 x 2 CTUs), every component on; SAO with one vertical and one horizontal virtual boundary."""
    rng = np.random.default_rng(5)
    W, H, ctu, bd = 64, 64, 32, 10
    k = dict(kind=kind, g=abi.make_geom(W, H, bd, ctu=ctu), planes=synth.noise_planes(rng, W, H, bd), vb=None, tables=None)
    if kind == "sao":
        k["ctus"] = synth.gen_sao(rng, W, H, ctu, bd, p_on=1.0)
        k["ctus"]["type"][0, 0] = 4
        v = abi.Vb(); v.numVer, v.numHor, v.posX[0], v.posY[0] = 1, 1, 24, 40
        k["vb"] = v
    else:
        t = synth.gen_alf(rng, W, H, ctu, bd, n_aps=2, n_cc=(2, 3))
        t["ctus"]["enable"][:] = 1
        t["ctus"]["ccIdx"][:] = 0
        k["tables"] = t; k["ctus"] = t["ctus"]
    return k


def _geom(**kw):
    def f(k):
        for n, v in kw.items():
            if n == "stride":
                for c in range(3): k["g"].stride[c] = v[c]
            else: setattr(k["g"], n, v)
    return f


def _rec(i, field, value, idx=None):
    def f(k):
        if idx is None: k["ctus"][field][i] = value
        else: k["ctus"][field][i, idx] = value
    return f


def _both(*edits):
    def f(k):
        for e in edits: e(k)
    return f


def _vb(**kw):
    def f(k):
        for n, v in kw.items():
            if n in ("posX", "posY"):
                for j, p in enumerate(v): getattr(k["vb"], n)[j] = p
            else: setattr(k["vb"], n, v)
    return f


def _tab(key, fn):
    def f(k):
        if key == "cc0": k["tables"]["cc"][0] = fn(k["tables"]["cc"][0])
        else: k["tables"][key] = np.ascontiguousarray(fn(k["tables"][key]))
    return f


_GEOM_ROWS = [
    ("chromaFormat 2", _geom(chromaFormat=2), _geom(chromaFormat=1)), ("chromaFormat 3", _geom(chromaFormat=3), _geom(chromaFormat=0)),
    ("CTU size 16", _geom(ctuSize=16), _geom(ctuSize=32)), ("CTU size 256", _geom(ctuSize=256), _geom(ctuSize=64)),
    ("bit depth 7", _geom(bitDepth=7), _geom(bitDepth=10)),
    ("width not a multiple of 8", _geom(width=60), _geom(width=64)), ("height not a multiple of 8", _geom(height=60), _geom(height=56)),
    ("luma stride below the width", _geom(stride=(60, 32, 32)), _geom(stride=(64, 32, 32))),
    ("luma stride not a multiple of 4", _geom(stride=(66, 32, 32)), _geom(stride=(68, 32, 32))),
    ("Cb stride below the width", _geom(stride=(64, 28, 32)), _geom(stride=(64, 32, 32))),
    ("Cr stride not a multiple of 4", _geom(stride=(64, 32, 34)), _geom(stride=(64, 32, 36))),
]
# (filter, what, edit that breaks a rule, the same edit with the offending field fixed)
REFUSALS = [("sao",) + r for r in _GEOM_ROWS] + [("alf",) + r for r in _GEOM_ROWS] + [
    ("sao", "bit depth 13", _geom(bitDepth=13), _geom(bitDepth=12)),
    ("sao", "type 5", _rec(1, "type", 5, 0), _rec(1, "type", 4, 0)), ("sao", "Cr type 254", _rec(2, "type", 254, 2), _rec(2, "type", 255, 2)),
    ("sao", "band 32", _both(_rec(0, "type", 4, 1), _rec(0, "band", 32, 1)), _both(_rec(0, "type", 4, 1), _rec(0, "band", 31, 1))),
    ("sao", "4 vertical VBs", _vb(numVer=4, posX=(8, 16, 40)), _vb(numVer=3, posX=(8, 16, 40))),
    ("sao", "-1 horizontal VBs", _vb(numHor=-1), _vb(numHor=0)),
    ("sao", "VB off the 8 grid", _vb(posX=(12,)), _vb(posX=(16,))), ("sao", "VB at x = 0", _vb(posX=(0,)), _vb(posX=(8,))),
    ("sao", "VB at x = W", _vb(posX=(64,)), _vb(posX=(56,))), ("sao", "VB at y = 4", _vb(posY=(4,)), _vb(posY=(8,))),
    ("alf", "bit depth 11", _geom(bitDepth=11), _geom(bitDepth=10)), ("alf", "bit depth 12", _geom(bitDepth=12), _geom(bitDepth=10)),
    ("alf", "15 luma sets", _both(_tab("lumaCoeff", lambda a: a[:15]), _tab("lumaClip", lambda a: a[:15]), _rec(slice(None), "lumaSet", 3)),
     _both(_tab("lumaCoeff", lambda a: a[:16]), _tab("lumaClip", lambda a: a[:16]), _rec(slice(None), "lumaSet", 3))),
    ("alf", "25 luma sets", _both(_tab("lumaCoeff", lambda a: np.concatenate([a, a[:7]])), _tab("lumaClip", lambda a: np.concatenate([a, a[:7]]))),
     _both(_tab("lumaCoeff", lambda a: np.concatenate([a, a[:6]])), _tab("lumaClip", lambda a: np.concatenate([a, a[:6]])))),
    ("alf", "lumaSet = numLumaSets", _rec(2, "lumaSet", 18), _rec(2, "lumaSet", 17)),
    ("alf", "lumaSet 200 with luma on", _rec(1, "lumaSet", 200), _both(_rec(1, "lumaSet", 200), _rec(1, "enable", 0, 0))),
    ("alf", "chromaAlt = numChromaAlts", _rec(3, "chromaAlt", 3, 1), _rec(3, "chromaAlt", 2, 1)),
    ("alf", "no chroma alternatives with chroma on", _both(_tab("chromaCoeff", lambda a: a[:0]), _tab("chromaClip", lambda a: a[:0])),
     _both(_tab("chromaCoeff", lambda a: a[:0]), _tab("chromaClip", lambda a: a[:0]), _rec(slice(None), "enable", 0, 1), _rec(slice(None), "enable", 0, 2))),
    ("alf", "ccIdx past numCc", _rec(0, "ccIdx", 3, 0), _rec(0, "ccIdx", 2, 0)),
    ("alf", "luma enable bit 7", _rec(0, "enable", 0x81, 0), _rec(0, "enable", 0x41, 0)),
    ("alf", "chroma enable bit 2", _rec(3, "enable", 5, 1), _rec(3, "enable", 3, 1)),
    ("alf", "PAD_TL with CLIP_TOP", _rec(3, "enable", 1 | 32 | 2, 0), _rec(3, "enable", 1 | 32 | 4, 0)),
    ("alf", "PAD_TL with CLIP_LEFT", _rec(3, "enable", 1 | 32 | 8, 0), _rec(3, "enable", 1 | 32 | 16, 0)),
    ("alf", "PAD_TL on the first CTU row", _rec(1, "enable", 1 | 32, 0), _rec(3, "enable", 1 | 32, 0)),
    ("alf", "PAD_TL on the first CTU column", _rec(2, "enable", 1 | 32, 0), _rec(2, "enable", 1 | 2, 0)),
    ("alf", "PAD_BR with CLIP_RIGHT", _rec(0, "enable", 1 | 64 | 16, 0), _rec(0, "enable", 1 | 64 | 8, 0)),
    ("alf", "PAD_BR with CLIP_BOTTOM", _rec(0, "enable", 1 | 64 | 4, 0), _rec(0, "enable", 1 | 64 | 2, 0)),
    ("alf", "PAD_BR on the last CTU column", _rec(1, "enable", 1 | 64, 0), _rec(0, "enable", 1 | 64, 0)),
    ("alf", "PAD_BR on the last CTU row", _rec(2, "enable", 1 | 64, 0), _rec(2, "enable", 1 | 16, 0)),
    ("alf", "PAD_WIDE with CC-ALF", _both(_rec(1, "ccIdx", 1, 1), _rec(1, "enable", 3, 2)), _both(_rec(1, "ccIdx", 0, 1), _rec(1, "enable", 3, 2))),
]


def refusal_variant(kind, edit):
    """The base call with one edit applied (copies of everything the edits touch); planes are widened to the edited strides."""
    k = refusal_base(kind)
    g = abi.Geom(); g.width, g.height, g.chromaFormat, g.bitDepth, g.ctuSize = k["g"].width, k["g"].height, k["g"].chromaFormat, k["g"].bitDepth, k["g"].ctuSize
    for c in range(3): g.stride[c] = k["g"].stride[c]
    k["g"] = g
    edit(k)
    if kind == "alf": k["ctus"] = k["tables"]["ctus"]
    k["planes"] = [np.ascontiguousarray(np.pad(p, ((0, 0), (0, max(0, k["g"].stride[c] - p.shape[1]))), constant_values=-7)) for c, p in enumerate(k["planes"])]
    return k


@pytest.mark.parametrize("kind,what,bad,fixed", REFUSALS, ids=[f"{r[0]}: {r[1]}" for r in REFUSALS])
def test_rule_rows(kind, what, bad, fixed):
    """The library refuses each edit, naming the entry point, and accepts it with the offending field fixed."""
    base = refusal_base(kind)
    assert synth.k45_record_problems(kind, base["g"], base["ctus"], base["tables"], base["vb"]) == []
    for edit, legal in ((bad, False), (fixed, True)):
        k = refusal_variant(kind, edit)
        probs = synth.k45_record_problems(kind, k["g"], k["ctus"], k["tables"], k["vb"])
        assert (probs == []) == legal, (what, legal, probs)
        assert legal or f"b200_{kind}_picture" in probs[0], (what, probs)
