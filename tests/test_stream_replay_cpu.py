"""The replay corpus on the CPU: every picture of real parsed streams (tests/stream_util.py corpus_names: the stream cases at two seeds, three geometries in
one stream, 200 fuzz draws), captured as the glue hands it to the device, replayed on its own through the oracle chain.

A record holds the picture's flattened lists, its geometry and copies of the DPB slots its PUs reference, taken before the picture is reconstructed.  If
replaying it from that snapshot alone gives the stock decoder's frame, the records are a complete statement of the picture, and tests/test_stream_replay_gpu.py
can hold the device to them: a difference there lies in a kernel or in picture.cu, not in the parser, the flattener or this harness."""
import collections, os, numpy as np, pytest
from oracle import vvc_stream as vs
from tests import helpers, stream_util as su
from vvdec_b200 import abi, synth

pytestmark = pytest.mark.skipif(not (vs.available() and os.path.exists(vs.SWAP_SO)), reason="oracle/_ref not built")


def ciip_blocks(pus, it):
    """luma intra records with a CIIP weight that sit on a PU (the inter half of a CIIP CU)"""
    at = set(zip(pus["x"].tolist(), pus["y"].tolist()))
    return sum((x, y) in at for x, y, c, w in zip(it["x"].tolist(), it["y"].tolist(), it["comp"].tolist(), it["ciip"].tolist()) if c == 0 and w > 0)


def coverage(rec, tiles):
    """What one captured picture exercises, counted from its lists and geometry (names of COVERAGE)"""
    g, pic = rec["geom"], rec["pic"]; f = pic["struct"].flags
    pus, it = pic["pus"], pic.get("intraTus")
    mono = g.chromaFormat == 0
    hits = {"4:0:0": mono, "4:0:0 with LMCS": mono and bool(f & abi.PIC_LMCS), "4:0:0 with ALF": mono and bool(f & abi.PIC_ALF), "8 bit": g.bitDepth == 8,
            f"CTU {g.ctuSize}": True, "width not a multiple of the CTU": g.width % g.ctuSize != 0, "height not a multiple of the CTU": g.height % g.ctuSize != 0,
            "chroma width 4 mod 8": not mono and (g.width >> 1) % 8 == 4, "tiles": tiles, "3 or more slices": len(pic.get("lfSlices", ())) >= 3,
            "scaling lists": "scaling" in pic, "weighted prediction": "wp" in pic, "LADF": "lfSeq" in pic and bool(pic["lfSeq"].ladfEnabled),
            "LMCS with chroma scaling": bool(f & abi.PIC_LMCS) and bool(pic["lmcs"]["struct"].chromaAdj),
            "CC-ALF": bool(f & abi.PIC_ALF) and bool((pic["alf"]["ctus"]["ccIdx"] > 0).any()),
            "GEO": bool((pus["flags"] & synth.PU_GEO).any()), "affine": bool((pus["flags"] & synth.PU_AFFINE).any()),
            "DMVR": bool((pus["flags"] & synth.PU_DMVR).any()), "BDOF": bool((pus["flags"] & synth.PU_BDOF).any()),
            "ISP": it is not None and bool((it["flags"] & abi.INTRA_ISP).any()), "CIIP": it is not None and ciip_blocks(pus, it) > 0,
            "intra list, CTU-resident K6 under auto": it is not None and helpers.intra_dense(g, len(it)),
            "intra list, one-CTA-per-block K6 under auto": it is not None and not helpers.intra_dense(g, len(it))}
    return [k for k, v in hits.items() if v]


COVERAGE = ["4:0:0", "4:0:0 with LMCS", "4:0:0 with ALF", "8 bit", "CTU 32", "CTU 64", "CTU 128", "width not a multiple of the CTU",
            "height not a multiple of the CTU", "chroma width 4 mod 8", "tiles", "3 or more slices", "scaling lists", "weighted prediction", "LADF",
            "LMCS with chroma scaling", "CC-ALF", "ISP", "CIIP", "GEO", "affine", "DMVR", "BDOF",
            "intra list, CTU-resident K6 under auto", "intra list, one-CTA-per-block K6 under auto"]


def selfcheck(name):
    """Worker: capture the stream, replay every picture through the oracle from its snapshot, compare with the stock frame of the picture (luma only for
    4:0:0) and with the DMVR deltas of the capture.  Returns the stream's mismatches and coverage."""
    cap = su.capture(name, su._WORKER_ORACLE)
    bad, hits = [], collections.Counter()
    for rec in cap["records"]:
        got, dm = su.oracle_replay(su._WORKER_ORACLE, rec)
        n = su.num_planes(rec["geom"])
        why = su.describe_difference(rec["pic"], got, cap["stock"][rec["frame"]], n)
        if why is None and not np.array_equal(dm, rec["dmvr"]): why = "DMVR deltas differ"
        if why: bad.append(f"{name} POC {rec['poc']}: {why}")
        hits.update(coverage(rec, cap["tiles"]))
    return dict(name=name, pictures=len(cap["records"]), bad=bad, hits=hits)


@pytest.fixture(scope="module")
def corpus():
    names = su.corpus_names()
    pool = su.CapturePool(names, selfcheck)
    try: return [pool.get(n) for n in names]
    finally: pool.close()


def test_corpus_size():
    names = su.corpus_names()
    assert len(names) == len(set(names)) and len(names) >= 280


def test_every_picture_replays_to_the_stock_frame(corpus):
    """The harness check: each captured picture, replayed from its snapshot alone (every other slot holds a sentinel picture), is the stock decoder's frame."""
    bad = [b for r in corpus for b in r["bad"]]
    assert not bad, f"{len(bad)} pictures differ; first: {bad[:3]}"
    assert sum(r["pictures"] for r in corpus) >= 1500


def test_corpus_coverage(corpus):
    """The corpus reaches the formats, geometries and tools the synthetic sweeps feed the device only in designed form."""
    hits = sum((r["hits"] for r in corpus), collections.Counter())
    missing = [k for k in COVERAGE if hits[k] == 0]
    assert not missing, (missing, dict(hits))
    assert hits["4:0:0"] >= 20 and hits["8 bit"] >= 100 and hits["tiles"] >= 20 and hits["chroma width 4 mod 8"] >= 100, dict(hits)


@pytest.fixture(scope="module")
def one_stream(oracle):
    return su.capture("gop_alf_ccalf-s1", oracle)


def test_a_perturbed_list_is_caught(oracle, one_stream):
    """The comparison has teeth: one TU level, or the coefficients of one ALF luma set, changed in a captured picture make the replay differ from the stock
    frame; restored, it agrees again."""
    rec = next(r for r in one_stream["records"] if r["pic"]["struct"].flags & abi.PIC_ALF and len(r["pic"]["tus"]))
    pic, stock = rec["pic"], one_stream["stock"][rec["frame"]]
    assert su.describe_difference(pic, su.oracle_replay(oracle, rec)[0], stock, 3) is None
    tus, coefs = pic["tus"], pic["coefs"]
    k = int(next(t for t in tus if t["comp"] == 0)["coefOff"]); old = int(coefs[k])               # the first level of the first luma TU
    coefs[k] = old + (64 if old <= 0 else -64)
    try: why = su.describe_difference(pic, su.oracle_replay(oracle, rec)[0], stock, 3)
    finally: coefs[k] = old
    assert why is not None and why.startswith("plane 0") and "tus" in why
    ctus = pic["alf"]["ctus"]; on = np.flatnonzero(ctus["enable"][:, 0])
    assert len(on)
    luma = pic["alfArrays"]["lumaCoeff"].reshape(-1, 1300); s = int(ctus["lumaSet"][on[0]])
    assert 0 <= s < len(luma)
    keep = luma[s].copy(); luma[s] = np.where(keep > 0, keep - 1, keep + 1)
    try: why = su.describe_difference(pic, su.oracle_replay(oracle, rec)[0], stock, 3)
    finally: luma[s] = keep
    assert why is not None
    assert su.describe_difference(pic, su.oracle_replay(oracle, rec)[0], stock, 3) is None


def test_covering_records_name_the_block_of_a_sample(one_stream):
    """The lookup a replay failure names its records with (shared with tools/stream_diag.py): every PU it returns covers the sample, and so does each TU."""
    rec = one_stream["records"][1]; pic = rec["pic"]
    for c, y, x in ((0, 37, 101), (1, 20, 50), (0, pic["pus"]["y"][-1], pic["pus"]["x"][-1])):
        r = su.covering_records(pic, c, int(y), int(x))
        X, Y = (x, y) if c == 0 else (2 * x, 2 * y)
        assert len(r["pus"]) + len(r.get("intra", ())) >= 1
        for p in r["pus"]: assert p["x"] <= X < p["x"] + p["w"] and p["y"] <= Y < p["y"] + p["h"]
        for t in r["tus"]:
            sc = 1 if t["comp"] == 0 else 2
            assert t["x"] * sc <= X < (t["x"] + (1 << t["log2w"])) * sc and t["y"] * sc <= Y < (t["y"] + (1 << t["log2h"])) * sc
