"""The designed K3 sweep (synth.lf_sweep) on the CPU: its grids are legal for the flat pass, every designed segment takes the decision it was built
for with its thresholds where they were put, the oracle changes only samples the classified decisions may write, and the sweep as a whole covers
every decision with every threshold on both sides.  Also: b200_lf_deblock, asked through synth.lf_grid_problems / lf_problems (its checks all run on the
host), accepts the golden grids and gen_lf_grid's, and refuses each row of the refusal table (tests/test_k3_gpu.py runs the accepted calls)."""
import os
import numpy as np
import pytest
from vvdec_b200 import abi, synth
from tests.helpers import lf_oracle, ROOT

CASES = list(synth.LF_SWEEP_CASES)


def _records(oracle, case):
    """Classified segments of both directions: vertical on the input, horizontal on the oracle's vertical-only output; and that output."""
    v = lf_oracle(oracle, case, 1)
    recs = {}
    for d, start in ((0, case["planes"]), (1, v)):
        for r in synth.lf_decisions(start, case["lfH" if d else "lfV"], d, case["g"], case["slices"], case["seq"], case["ctuSlice"]):
            recs[(r["dir"], r["comp"], r["x"], r["y"])] = r
    return recs, v


@pytest.mark.parametrize("name", CASES)
def test_sweep_grids_are_legal(name):
    case = synth.lf_sweep(name)
    for d in (0, 1):
        assert synth.lf_grid_problems(case["lfH" if d else "lfV"], d, case["g"]) == [], (name, d)


@pytest.mark.parametrize("name", [n for n in CASES if synth.lf_sweep(n)["classify"]])
def test_designed_decisions_and_footprints(oracle, name):
    """Every designed segment takes its tag and meets its probes; per direction, every sample the oracle changes lies in the footprint of a classified
    decision; 'none' / 'off' segments keep their samples, every designed segment whose decision filters changes one (in the block pictures:
    every segment with tc > 0).  In the tight-spacing and geometry pictures every luma edge filters, both directions."""
    case = synth.lf_sweep(name)
    recs, v = _records(oracle, case)
    for s in case["segs"]:
        r = recs[(s["dir"], s["comp"], s["x"], s["y"])]
        where = f"{name}: {'H' if s['dir'] else 'V'} comp {s['comp']} ({s['x']}, {s['y']})"
        assert s["tag"] in ("any", r["tag"]), (where, s["tag"], r["tag"], r["q"])
        for qn, tn, off in s["probes"]:
            assert r["q"][qn] - r["q"][tn] == off, (where, qn, tn, off, r["q"][qn], r["q"][tn])
    out = lf_oracle(oracle, case, 3)
    for d, before, after in ((0, case["planes"], v), (1, v, out)):
        for c in range(3 if case["chroma"] else 1):
            mine = [r for r in recs.values() if r["dir"] == d and r["comp"] == c]
            allowed = set().union(*[r["writes"] for r in mine]) if mine else set()
            changed = {tuple(p) for p in np.argwhere(before[c] != after[c]).tolist()}
            assert changed <= allowed, (name, d, c, sorted(changed - allowed)[:4])
            must = {(s["x"], s["y"]) for s in case["segs"] if s["dir"] == d and s["comp"] == c and s["tag"] != "any"} if case["segs"] else None
            for r in mine:
                if r["tag"] in ("none", "none_ctb", "off", "weak_cut"):
                    assert not (r["writes"] & changed), (name, d, c, r["x"], r["y"], r["tag"])
                elif r["q"]["tc"] and (must is None or (r["x"], r["y"]) in must):   # designed segments, and every edge of the block pictures
                    assert r["writes"] & changed, (name, d, c, r["x"], r["y"], r["tag"], "filters but changes nothing")
    if name == "tight_spacing" or name.startswith("geometry"):
        luma = [r for r in recs.values() if r["comp"] == 0]
        assert luma and all(r["tag"] not in ("none", "weak_cut") for r in luma), (name, sorted({r["tag"] for r in luma}))


LUMA_TAGS = {"none", "weak_cut", "weak00", "weak01", "weak10", "weak11", "strong"} | {f"long{p}{q}" for p in (3, 5, 7) for q in (3, 5, 7) if (p, q) != (3, 3)}
CHROMA_TAGS = {f"{t}{s}" for t in ("none", "chroma_weak_small", "chroma_weak_d", "chroma_weak", "chroma_strong") for s in ("", "_ctb")}


def test_sweep_covers_every_decision_and_threshold(oracle):
    """Across the designed cases: every luma and chroma tag appears as a designed segment in both directions (chroma CTB forms: horizontal only), at
    CTU 32, 64 and 128 for the CTB forms, and every (quantity, threshold) probe appears on both sides of its threshold.  The clipping case reaches the
    [0, pmax] clip of the weak filter."""
    seen, sides, ctb_ctus = set(), {}, set()
    for name in CASES:
        case = synth.lf_sweep(name)
        for s in case["segs"]:
            seen.add((s["tag"], s["dir"]))
            if s["tag"].endswith("_ctb"): ctb_ctus.add(case["ctu"])
            for qn, tn, off in s["probes"]: sides.setdefault((qn[:-2] if qn[-2] == "_" else qn, tn), set()).add(off >= 0)
    for t in LUMA_TAGS | {t for t in CHROMA_TAGS if not t.endswith("_ctb")}:
        assert (t, 0) in seen and (t, 1) in seen, t
    for t in CHROMA_TAGS:
        if t.endswith("_ctb"): assert (t, 1) in seen, t
    assert ctb_ctus >= {32, 64, 128}
    assert {k for k, v in sides.items() if v != {True, False}} == set(), sides
    assert {("dsum", "beta"), ("adelta", "thrCut"), ("adelta", "tc"), ("pside", "sideThr"), ("qside", "sideThr"), ("d2", "beta2"), ("pq", "tc25"),
            ("s", "beta3"), ("d2L", "beta4"), ("sL", "beta35")} <= set(sides)
    recs, _ = _records(oracle, synth.lf_sweep("clipping_12bit"))
    assert any(r["q"].get("clip01") for r in recs.values())


def test_sweep_reaches_qp_extremes():
    """tc index 0 and 65 (clipped), beta index 0 and 63, QP -24 at 12 bit and offsets of +-12 appear in the qp cases; the LADF cases have 5 intervals and
    luma levels on every lower bound and one above it."""
    for bd in (8, 9, 10, 12):
        case = synth.lf_sweep(f"qp_extremes_{bd}bit")
        qps = case["lfV"]["qp"][..., 0][case["lfV"]["bs"] > 0]
        assert qps.min() == -6 * (bd - 8) and qps.max() == 63
        assert {12, -12} <= set(case["slices"]["tc"].ravel().tolist()) and {12, -12} <= set(case["slices"]["beta"].ravel().tolist())
    for bd in (10, 12):
        seq, pairs = synth._lf_ladf(bd)
        assert seq.ladfNumIntervals == 5
        levels = {lvl for lvl, qp in pairs}
        assert all({seq.ladfIntervalLowerBound[k], seq.ladfIntervalLowerBound[k] + 1} <= levels for k in range(1, 5))
        assert min(qp + seq.ladfQpOffset[k] for lvl, qp in pairs for k in range(5)) < 0


def test_rule_accepts_golden_and_generated_grids():
    z = np.load(os.path.join(ROOT, "tests", "golden", "k3_deblock_picture.npz"))
    W, H, bd, ctu = (int(v) for v in z["geom"])
    g = abi.make_geom(W, H, bd, ctu=ctu)
    for d, k in ((0, "lfV"), (1, "lfH")):
        assert synth.lf_grid_problems(z[k], d, g) == [], k
    for seed, W, H, ctu in [(1, 256, 128, 128), (2, 416, 240, 64), (3, 200, 136, 32), (4, 1920, 1080, 128), (7, 832, 480, 32)]:
        rng = np.random.default_rng(seed)
        cus = synth.partition(rng, W, H, ctu=ctu)
        lfV, lfH = synth.gen_lf_grid(rng, cus, W, H)
        g = abi.make_geom(W, H, 10, ctu=ctu)
        assert synth.lf_grid_problems(lfV, 0, g) == [] and synth.lf_grid_problems(lfH, 1, g) == [], seed


# ---- refusals: a small legal base picture and one edit per rule (the GPU file runs each through b200_lf_deblock)
def refusal_base():
    """64 x 64, 10 bit, 4:2:0, CTU 32: blocks 8, 8, 16, 32 in both directions (vertical edges at x = 8, 16 (3/3) and 32 (3/7))."""
    cv = synth._lf_block_case(synth._LfCanvas(64, 64, 10, 32), [8, 8, 16, 32], [8, 8, 16, 32], 12)
    case = cv.case("refusal_base")
    case["ctuSlice"] = np.zeros(4, np.uint8)
    case["dirs"] = 3
    return case


def _edge(d, x, y, P, Q, bs=2):
    def f(k):
        e = k["lfH" if d else "lfV"][y // 4, x // 4]
        e["bs"], e["len"] = bs, 128 + (P << 4) + Q
    return f


def _line(d, at, edges):
    """Replaces the luma edges of one line (row of lfV / column of lfH) by `edges`: (position, P, Q)."""
    def f(k):
        g = k["lfH" if d else "lfV"]
        ln = g[:, at // 4] if d else g[at // 4]
        ln["bs"] = 0; ln["len"] = 0
        for pos, P, Q in edges: ln[pos // 4]["bs"], ln[pos // 4]["len"] = 2, 128 + (P << 4) + Q
    return f


def _geom(**kw):
    def f(k):
        for n, v in kw.items():
            if n == "stride":
                for c in range(3): k["g"].stride[c] = v[c]
            else: setattr(k["g"], n, v)
    return f


def _set(n, v):
    def f(k): k[n] = v
    return f


def _cs(i, v):
    def f(k): k["ctuSlice"][i] = v
    return f


# (what, edit that breaks a rule, the same edit with the offending field fixed, whether it breaks a rule of the grid scan)
REFUSALS = [
    ("chromaFormat 2", _geom(chromaFormat=2), _geom(chromaFormat=1), False), ("chromaFormat 3", _geom(chromaFormat=3), _geom(chromaFormat=0), False),
    ("bit depth 7", _geom(bitDepth=7), _geom(bitDepth=8), False), ("bit depth 13", _geom(bitDepth=13), _geom(bitDepth=12), False),
    ("width not a multiple of 8", _geom(width=60), _geom(width=64), False), ("height not a multiple of 8", _geom(height=60), _geom(height=64), False),
    ("luma stride below the width", _geom(stride=(63, 32, 32)), _geom(stride=(64, 32, 32)), False),
    ("chroma stride below the width", _geom(stride=(64, 32, 31)), _geom(stride=(64, 32, 32)), False),
    ("dirs 4", _set("dirs", 4), _set("dirs", 2), False), ("dirs 7", _set("dirs", 7), _set("dirs", 3), False),
    ("ctuSlice past numSlices", _cs(3, 1), _cs(3, 0), False),
    ("luma length 0", _edge(0, 8, 8, 0, 3), _edge(0, 8, 8, 1, 1), True), ("luma length 4", _edge(0, 16, 20, 3, 4), _edge(0, 16, 20, 3, 3), True),
    ("luma length 6", _edge(1, 24, 8, 6, 3), _edge(1, 24, 8, 7, 3), True),
    ("luma Bs 3", _edge(0, 16, 0, 3, 3, bs=3), _edge(0, 16, 0, 3, 3, bs=2), True), ("chroma Bs 3", _edge(0, 16, 0, 3, 3, bs=2 | 3 << 4), _edge(0, 16, 0, 3, 3, bs=2 | 2 << 4), True),
    ("vertical edge on the first column", _edge(0, 0, 12, 3, 3), _edge(0, 0, 12, 3, 3, bs=0), True),
    ("horizontal edge on the first row", _edge(1, 40, 0, 3, 3, bs=2 << 2), _edge(1, 40, 0, 3, 3, bs=0), True),
    ("long Q side past the right border", _edge(0, 60, 4, 3, 7), _edge(0, 60, 4, 3, 3), True),
    ("long Q side past the bottom border", _edge(1, 4, 60, 3, 5), _edge(1, 4, 60, 3, 3), True),
    ("long P side before the first column", _line(0, 16, [(4, 5, 5), (16, 3, 3), (32, 3, 7)]), _line(0, 16, [(4, 3, 5), (16, 3, 3), (32, 3, 7)]), True),
    ("Q writes 2 where the next edge reads 3, 4 apart", _line(0, 24, [(8, 3, 2), (12, 1, 1), (32, 3, 3)]), _line(0, 24, [(8, 3, 1), (12, 1, 1), (32, 3, 3)]), True),
    ("Q reads 3 where the next edge writes 2, 4 apart", _line(1, 28, [(8, 3, 1), (12, 2, 1), (32, 3, 3)]), _line(1, 28, [(8, 3, 1), (12, 1, 1), (32, 3, 3)]), True),
]


def refusal_variant(edit):
    """The base case with one edit applied (copies of everything the edits touch)."""
    k = refusal_base()
    g = abi.Geom(); g.width, g.height, g.chromaFormat, g.bitDepth, g.ctuSize = k["g"].width, k["g"].height, k["g"].chromaFormat, k["g"].bitDepth, k["g"].ctuSize
    for c in range(3): g.stride[c] = k["g"].stride[c]
    k["g"] = g
    edit(k)
    return k


@pytest.mark.parametrize("what,bad,fixed,grid", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_rule_rows(what, bad, fixed, grid):
    """Every row of the refusal table: b200_lf_deblock refuses the edit, naming itself, and accepts it with the offending field fixed; a grid row is
    refused for its grid alone."""
    assert synth.lf_problems(refusal_base()) == []
    probs = synth.lf_problems(refusal_variant(bad))
    assert len(probs) == 1 and "b200_lf_deblock" in probs[0], (what, probs)
    assert synth.lf_problems(refusal_variant(fixed)) == [], what
    if grid:
        k = refusal_variant(bad)
        assert not all(synth.lf_grid_legal(k["lfH" if d else "lfV"], d, k["g"]) for d in (0, 1)), what
