"""The designed K2 sweep (synth.mc_sweep) reaches what tests/test_k2_gpu.py and tests/test_k2_oracle_vs_ref.py rely on (no device needed): every tile
list with every luma phase pair, every shape x tool pair, windows exactly at their interior / boundary thresholds, no overlapping PUs, and — through the
oracle — DMVR searches that end on each of the 25 integer positions, both sub-sample tie offsets, flat error surfaces and the early exit."""
import numpy as np
import pytest
from vvdec_b200 import synth
from tests import helpers

CASES = list(synth.MC_SWEEP_CASES)


@pytest.mark.parametrize("name", CASES)
def test_pus_are_legal_and_do_not_overlap(name):
    c = synth.mc_sweep(name)
    occ = np.zeros((c["H"], c["W"]), bool)
    for p in c["pus"]:
        x, y, w, h = int(p["x"]), int(p["y"]), int(p["w"]), int(p["h"])
        assert x % 4 == 0 and y % 4 == 0 and x + w <= c["W"] and y + h <= c["H"]
        assert x // c["ctu"] == (x + w - 1) // c["ctu"] and y // c["ctu"] == (y + h - 1) // c["ctu"], "a PU crosses a CTU boundary"
        assert not occ[y:y + h, x:x + w].any(), (name, p)
        occ[y:y + h, x:x + w] = True
    bi = (c["pus"]["refSlot"] >= 0).all(axis=1)
    dm = (c["pus"]["flags"] & synth.PU_DMVR) != 0
    assert not (dm & ~bi).any() and (c["bd"] <= 10 or not dm.any())
    assert (c["pus"]["refSlot"][dm] == np.stack([c["pus"]["refSlot"][dm][:, 0], c["pus"]["refSlot"][dm][:, 0] + 2], 1)).all()   # POC pairs (4, 12) and (0, 16)


def test_every_list_and_phase_pair():
    for name in ("phases_10bit", "phases_8bit_stride_odd"):
        c = synth.mc_sweep(name)
        seen = {}
        for i, tx, ty, lst in synth.mc_tiles(c["pus"]):
            p = c["pus"][i]
            l = 0 if p["refSlot"][0] >= 0 else 1
            seen.setdefault(lst, set()).add((int(p["mv"][l][0]) & 15, int(p["mv"][l][1]) & 15))
        want = [m * 4 + k for m, k in synth.MC_LISTS]
        assert all(len(seen.get(l, ())) == 256 for l in want), {l: len(seen.get(l, ())) for l in want}
    # every chroma 1/32 phase (x and y), the AltHpel half-sample ones among them
    c = synth.mc_sweep("phases_10bit")
    mv = c["pus"]["mv"][:, 0]
    assert set((mv[:, 0] & 31).tolist()) == set(range(32)) and set((mv[:, 1] & 31).tolist()) == set(range(32))
    alt = c["pus"][(c["pus"]["flags"] & synth.PU_ALTHPEL) != 0]
    assert {(int(a) & 31, int(b) & 31) for a, b in alt["mv"][:, 0]} == {(a, b) for a in (0, 8, 16, 24) for b in (0, 8, 16, 24)}
    # the affine list and every other list: every class of every mode is in the shapes case too
    lists = {lst for _, _, _, lst in synth.mc_tiles(synth.mc_sweep("shapes_10bit")["pus"])}
    assert lists == {m * 4 + k for m, k in synth.MC_LISTS} | {16}


def test_every_shape_and_tool():
    c = synth.mc_sweep("shapes_10bit")
    have = {(t, int(p["w"]), int(p["h"])) for t, p in zip(c["tags"], c["pus"])}
    for t in synth.MC_TOOLS:
        if t == "geo": continue
        for w in synth.MC_SIZES:
            for h in synth.MC_SIZES:
                if synth.mc_tool_legal(t, w, h): assert (t, w, h) in have, (t, w, h)
    geo = c["pus"][(c["pus"]["flags"] & synth.PU_GEO) != 0]
    assert sorted(geo["bcwW1"].tolist()) == list(range(64))
    assert {(int(p["w"]), int(p["h"])) for p in geo} == {(w, h) for w in synth.MC_SIZES for h in synth.MC_SIZES if synth.mc_tool_legal("geo", w, h)}
    assert set(c["pus"]["bcwW1"][(c["pus"]["flags"] & synth.PU_GEO) == 0].tolist()) == {-2, 3, 4, 5, 10}
    w = synth.mc_sweep("wp_10bit")
    assert set(synth.MC_WP_TOOLS) <= {t for t, p in zip(w["tags"], w["pus"]) if p["wpIdx"]} and (w["pus"]["wpIdx"] == 0).any()
    assert synth.mc_sweep("shapes_yuv400_10bit")["g"].chromaFormat == 0 and synth.mc_sweep("edges_ctu32_yuv400_8bit")["g"].chromaFormat == 0
    assert {synth.mc_sweep(n)["bd"] for n in synth.MC_SWEEP_CASES} == {8, 10, 12}
    assert any(synth.mc_sweep(n)["H"] % 16 for n in synth.MC_SWEEP_CASES)
    strides = [synth.mc_sweep(n)["strides"] for n in synth.MC_SWEEP_CASES]
    assert any(s[0] % 2 for s in strides) and any(s[0] % 2 == 0 and s[0] % 8 and s[0] != synth.mc_sweep(n)["W"] for s, n in zip(strides, synth.MC_SWEEP_CASES))


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("edges")])
def test_threshold_tiles_sit_on_their_threshold(name):
    c = synth.mc_sweep(name)
    g = c["g"]
    hit, special = set(), set()
    for i, kind, edge, off, l in c["marks"]:
        p = c["pus"][i]
        if kind in ("clip", "far"): special.add((kind, edge)); continue
        w, h = int(p["w"]), int(p["h"])
        assert w <= 16 and h <= 16                                                  # one tile: its window is the PU's
        x0, x1, y0, y1 = synth.mc_window_margins(kind, g.width, g.height, w, h)
        x, y = synth.mc_tile_windows(p, l)[kind]
        want = {"l": x0, "r": x1, "t": y0, "b": y1}[edge] + off
        assert (x if edge in "lr" else y) == want, (i, kind, edge, off)
        hit.add((synth.mc_list_of(p, 0, 0), kind, edge, off))
    kinds_per_mode = {3: ["dmvr"] + (["dmvr_chroma"] if c["chroma"] else [])}
    for m, k in synth.MC_LISTS:
        if m == 3 and c["bd"] > 10: continue
        for kind in kinds_per_mode.get(m, ["luma"] + (["chroma"] if c["chroma"] else [])):
            assert all((m * 4 + k, kind, e, o) in hit for e in "lrtb" for o in (-1, 0, 1)), (m, k, kind)
    # DMVR tiles: the search window is fast only when every list's luma and chroma origins are interior (k2_inter.cu dmvr_search).  Where all the other
    # conditions hold, the marked origin decides the path; in 4:2:0 the chroma condition is the stricter one (icx >= 4 needs ix >= 8), so a luma threshold
    # tile whose chroma origin is outside takes the slow path anyway: only the 4:0:0 cases make the luma DMVR thresholds path boundaries
    even = all(st % 2 == 0 for st in c["strides"][:3 if c["chroma"] else 1])
    decisive = set()
    for i, kind, edge, off, l in c["marks"]:
        if not kind.startswith("dmvr") or not even: continue
        p = c["pus"][i]; w, h = int(p["w"]), int(p["h"])
        inside = {}
        for ll in range(2):
            win = synth.mc_tile_windows(p, ll)
            for k in ("dmvr", "dmvr_chroma")[:2 if c["chroma"] else 1]:
                x0, x1, y0, y1 = synth.mc_window_margins(k, g.width, g.height, w, h)
                inside[ll, k] = x0 <= win[k][0] <= x1 and y0 <= win[k][1] <= y1
        fast = all(inside.values())
        if all(v for key, v in inside.items() if key != (l, kind)):
            assert fast == inside[l, kind] == (off <= 0 if edge in "rb" else off >= 0), (i, kind, edge, off)
            decisive.add((kind, edge, off))
        else:
            assert not fast and (not inside[l, kind] or (kind == "dmvr" and c["chroma"])), (i, kind, edge, off)
    if even:
        want = {(k, e, o) for k in (("dmvr_chroma",) if c["chroma"] else ("dmvr",)) for e in "lrtb" for o in ((0, -1) if e in "rb" else (0, 1))}   # on / just inside
        assert want <= decisive or c["bd"] > 10, sorted(want - decisive)
    # MVs at each clipMv bound and one sample past it (PUs of every size up to the CTU), and near +-2^17
    assert {e for k, e in special if k == "clip"} == {"xlo", "xlo-1", "xhi", "xhi+1", "ylo", "ylo-1", "yhi", "yhi+1"}
    assert {e for k, e in special if k == "far"} == {"+", "-"}
    for i, kind, edge, _, _ in c["marks"]:
        if kind == "clip":
            p = c["pus"][i]; ax = 0 if edge[0] == "x" else 1; pos = int(p["x"] if ax == 0 else p["y"])
            S = g.width if ax == 0 else g.height
            lo, hi = (-c["ctu"] - 8 - pos + 1) * 16, (S + 8 - pos - 1) * 16
            v = int(p["mv"][0][ax])
            assert (lo <= v < lo + 16) if edge.endswith("lo") else (lo - 16 <= v < lo) if edge.endswith("lo-1") else (hi <= v < hi + 16) if edge.endswith("hi") else v >= hi + 16


def test_affine_spreads_straddle_the_limit():
    for name in ("affine_limits_10bit", "affine_limits_12bit_stride_odd"):
        c = synth.mc_sweep(name)
        over = {(bool(p["flags"] & synth.PU_AFFINE6), int(p["interDir"]) == 3, synth.mc_affine_over(p, 0 if p["refSlot"][0] >= 0 else 1)) for p in c["pus"]}
        assert over == {(six, bi, o) for six in (False, True) for bi in (False, True) for o in (False, True)}   # 4- / 6-parameter, uni / bi, under / over
        eq = [p for p in c["pus"] if (p["cpmv"][0] == p["mv"][0]).all() and (p["cpmv"][1] == p["mv"][1]).all()]
        assert len(eq) >= 8                                                         # equal CPMVs: PROF off whatever the flag says


def test_far_mvs(oracle):
    """MVs near +-2^17: the affine sub-block MVs pass the storage clamp; DMVR from such MVs searches border replicas only and ends at the centre (zero
    delta), so its refinement never crosses the clamp."""
    c = synth.mc_sweep("edges_ctu128")
    _, dm = helpers.mc_oracle(oracle, c)
    far = [c["pus"][i] for i, kind, *_ in c["marks"] if kind == "far"]
    for p in far:
        if p["flags"] & synth.PU_DMVR: assert (dm[int(p["dmvrOff"])] == 0).all()
        if p["flags"] & synth.PU_AFFINE:
            LT, dHX = int(p["mv"][0][0]), (int(p["cpmv"][0][0][0]) - int(p["mv"][0][0])) << (7 - (int(p["w"]).bit_length() - 1))
            assert abs((LT * 128 + dHX * (2 + 4 * (int(p["w"]) // 4 - 1))) >> 7) > (1 << 17)
    assert any(p["flags"] & synth.PU_DMVR for p in far) and any(p["flags"] & synth.PU_AFFINE for p in far)


def _dmvr_deltas(oracle, name):
    c = synth.mc_sweep(name)
    _, dm = helpers.mc_oracle(oracle, c)
    return c, dm


def test_dmvr_reaches_every_position(oracle):
    """The mirrored search ends on each of the 25 integer positions (the +-2 rows and columns without the sub-sample surface), the centre ones by the
    early exit; all sub-blocks of a PU agree."""
    for name in ("dmvr_targets_10bit", "dmvr_targets_8bit_stride_pad"):
        c, dm = _dmvr_deltas(oracle, name)
        reached = set()
        for i, u, v in c["targets"]:
            p = c["pus"][i]
            n = max(1, int(p["w"]) >> 4) * max(1, int(p["h"]) >> 4)
            d = dm[int(p["dmvrOff"]):int(p["dmvrOff"]) + n]
            for q, t in ((d[:, 0], u), (d[:, 1], v)):
                if abs(t) == 2: assert (q == 16 * t).all(), (name, i, u, v, d.tolist())
                else: assert (abs(q - 16 * t) <= 8).all(), (name, i, u, v, d.tolist())
            if u == 0 and v == 0: assert (d == 0).all()                              # SAD 0 at the centre: the early exit
            reached.add((u, v))
        assert reached == {(u, v) for u in range(-2, 3) for v in range(-2, 3)}


def test_dmvr_designed_surfaces(oracle):
    """Designed cost surfaces (synth.MC_DMVR_SURFACES): a neighbour equal to the scaled centre cost gives the -8 / +8 tie offsets, two equal neighbours
    a zero denominator, identical flat windows the early exit.  bioAppliedSubblk is not exported: den0_x_bio_off, den0_x_ramp_y_bio_off (minCost 1.5 * tw * th) and
    flat_exit / the targets case (minCost 0) stand for BDOF switched off in a DMVR sub-block, den0_x / the tie cases (minCost >= 3 * tw * th) for it on."""
    c, dm = _dmvr_deltas(oracle, "dmvr_surfaces_10bit")
    for p, kind in zip(c["pus"], c["tags"]):
        n = max(1, int(p["w"]) >> 4) * max(1, int(p["h"]) >> 4)
        d = dm[int(p["dmvrOff"]):int(p["dmvrOff"]) + n]
        assert (d == np.array(synth.MC_DMVR_SURFACES[kind])).all(), (kind, p, d.tolist())
