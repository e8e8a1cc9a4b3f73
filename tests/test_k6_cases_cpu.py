"""The K6 test lists reach what tests/test_k6_intra_gpu.py claims they reach (no device needed): the designed sweep holds every block it lists and no
block of it reads another, and the generated cases put more than 1024 records into one CTU, stay below the density threshold where they stand for a B
picture, and never use MRL on the first row of a CTU."""
import numpy as np
import pytest
from vvdec_b200 import abi, synth
from tests import helpers


def test_designed_sweep_covers_its_list():
    W, H, recs = synth.intra_sweep()
    want = set(synth.intra_sweep_blocks())
    keys = [synth.intra_record_key(r) for r in recs]
    assert set(keys) == want
    # every block once per neighbourhood: full (the straight-copy fetch), partial (substitution), none
    full = {k for k, r in zip(keys, recs) if r["flags"] & abi.INTRA_AVAIL_TL}
    unit = np.where(recs["comp"] > 0, 2, 4)
    n_full = 2 * (1 << recs["log2w"].astype(int)) // unit + 2 * (1 << recs["log2h"].astype(int)) // unit
    total = recs["numAbove"].astype(int) + recs["numLeft"].astype(int)
    assert full == want and len(recs) == 3 * len(want)
    assert np.array_equal((recs["flags"] & abi.INTRA_AVAIL_TL) != 0, total == n_full)
    assert {k for k, t in zip(keys, total) if t == 0} == want
    partial = [(k, r) for k, r, t, n in zip(keys, recs, total, n_full) if 0 < t < n]
    assert {k for k, _ in partial} == want
    assert any(r["numAbove"] < 2 * (1 << int(r["log2w"])) // (2 if r["comp"] else 4) for _, r in partial)
    assert any(r["numLeft"] < 2 * (1 << int(r["log2h"])) // (2 if r["comp"] else 4) for _, r in partial)
    # shapes, modes and wide-angle remaps
    luma = {(w, h) for (c, w, h, *_) in want if c == 0}
    chroma = {(c, w, h) for (c, w, h, *_) in want if c}
    assert len(luma) == 25 and len(chroma) == 32
    for c, w, h in [(0, w, h) for (w, h) in luma] + sorted(chroma):
        assert all((c, w, h, m, 0, 0) in want for m in range(67))
        for m in range(2, 67):
            if synth.intra_wide_angle(w, h, m) != m: assert (c, w, h, m, 0, 0) in want
    remaps = {(w, h, m) for (c, w, h, m, mrl, mip) in want if m <= 66 and synth.intra_wide_angle(w, h, m) != m}
    assert len(remaps) > 100
    assert all((0, w, h, m, mrl, 0) in want for (w, h) in luma for mrl in (1, 2) for m in range(2, 67))
    assert all((0, w, h, abi.INTRA_MIP, 0, k | (t << 7)) in want for (w, h) in luma for t in (0, 1)
               for k in range(16 if (w, h) == (4, 4) else 8 if (w == 4 or h == 4 or (w, h) == (8, 8)) else 6))
    assert any(r["flags"] & abi.INTRA_FILTER_REF for r in recs)


def test_designed_sweep_is_independent_and_in_ctu_order():
    """No block's reference samples (row above incl. above-right and the corner, column left incl. below-left, MRL lines) are samples of another block:
    the sweep has no dependencies.  Records are in CTU raster order, every block inside its CTU."""
    W, H, recs = synth.intra_sweep()
    ctu = 128
    key = ((recs["y"].astype(np.int64) << (recs["comp"] > 0)) // ctu) * (W // ctu) + ((recs["x"].astype(np.int64) << (recs["comp"] > 0)) // ctu)
    assert np.all(np.diff(key) >= 0)
    for c in range(3):
        r = recs[recs["comp"] == c]
        pw, ph = (W, H) if c == 0 else (W // 2, H // 2)
        cs = ctu >> (1 if c else 0)
        occ = np.zeros((ph, pw), bool)
        for t in r:
            x, y, w, h = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"])
            assert x // cs == (x + w - 1) // cs and y // cs == (y + h - 1) // cs
            assert not occ[y:y + h, x:x + w].any()
            occ[y:y + h, x:x + w] = True
        for t in r:
            x, y, w, h, m = int(t["x"]), int(t["y"]), 1 << int(t["log2w"]), 1 << int(t["log2h"]), int(t["multiRefIdx"])
            assert x + 2 * w <= pw and y + 2 * h <= ph
            assert not occ[y - 1 - m:y, x - 1 - m:x + 2 * w].any() and not occ[y - 1 - m:y + 2 * h, x - 1 - m:x].any(), (c, x, y, w, h)


def test_generator_cases_reach_their_regime():
    counts = {}
    for name in ("ctu_1244_blocks", "ctu_1024_blocks", "sparse_1080p", "ctu64_200x136", "stride_420", "stride_417", "yuv400_8bit"):
        kw = helpers.INTRA_CASES[name]
        g, planes, resi, recs = helpers.intra_case(**kw)
        counts[name] = helpers.intra_ctu_counts(recs, kw["ctu"], kw["W"]).max()
        if name == "sparse_1080p":
            assert not helpers.intra_dense(g, len(recs))                          # v1 under auto
            assert set(np.unique(recs["ciip"][recs["ciip"] > 0]).tolist()) == {1, 2, 3}
        if name == "stride_420": assert all(s % 8 and not s % 2 for s in g.stride)
        if name == "stride_417": assert all(s % 2 for s in g.stride)
        if name == "yuv400_8bit": assert (recs["comp"] == 0).all() and planes[1] is None and g.chromaFormat == 0
        if name == "ctu64_200x136": assert ((recs["comp"] > 0) & (recs["x"] >= 96)).any() and ((recs["comp"] > 0) & (recs["y"] >= 64)).any()   # the 4-sample chroma tiles
    assert counts["ctu_1244_blocks"] > 1024                                          # records past the 1024 the CTU-resident kernel stages
    assert counts["ctu_1024_blocks"] == 1024


@pytest.mark.parametrize("ctu", [32, 64, 128])
def test_no_mrl_on_the_first_row_of_a_ctu(ctu):
    for seed in range(4):
        rng = np.random.default_rng(seed)
        layout = synth.gen_intra_layout(rng, 416, 240, ctu, min_size=4)
        recs = synth.gen_intra_records(rng, layout, 416, 240, p_mrl=0.5, ctu=ctu)
        mrl = recs[recs["multiRefIdx"] > 0]
        assert len(mrl) > 20 and not (mrl["y"] % ctu == 0).any()
