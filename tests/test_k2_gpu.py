"""K2 parity on the GPU: CUDA inter prediction (through the C ABI) vs the pinned oracle, bit-exact (samples and DMVR MV deltas), on random PU lists and on
every case of the designed sweep (synth.mc_sweep); and the wrapper's and the list validation's refusals."""
import ctypes as C
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth
from tests.helpers import ref_ptrs, mc_dst, mc_oracle, mc_mismatch
from tests.test_k2_oracle_vs_ref import _case

pytestmark = pytest.mark.gpu


def _compare(b200, oracle, case):
    """b200_mc_predict_wp against the oracle on one case (the dict of synth.mc_sweep): destinations start as a sentinel, so that a sample K2 does not
    write is caught as well as one it writes wrongly."""
    a, da = mc_oracle(oracle, case)
    g, pus = case["g"], case["pus"]
    b = mc_dst(g); db = np.zeros_like(da)
    ent = case["wp"][1] if case.get("wp") else None
    vvdec_b200.check(b200.b200_mc_predict_wp(C.byref(g), abi.plane_ptrs(b), ref_ptrs(case["refs"]), len(case["refs"]), pus.ctypes.data, len(pus), db.ctypes.data,
                                             len(db), None if ent is None else ent.ctypes.data, 0 if ent is None else len(ent)))
    msg = mc_mismatch(case, a, b, da, db)
    assert msg is None, msg


def _random_case(name, seed, W, H, bd, wp=False, **kw):
    pus, nd, refs = _case(seed, W, H, bd, **kw)
    case = dict(name=name, g=abi.make_geom(W, H, bd), W=W, H=H, bd=bd, chroma=1, strides=(W, W // 2, W // 2), pus=pus, ndmvr=nd, refs=refs,
                tags=["random"] * len(pus), wp=None)
    if wp: case["wp"] = synth.gen_wp(np.random.default_rng(seed), bd, pus)
    return case


@pytest.mark.parametrize("name,kw", [("regular", dict(p_dmvr=0, p_bdof=0, p_affine=0)), ("bdof", dict(p_dmvr=0, p_bdof=0.9, p_affine=0, p_bi=0.9)),
                                      ("dmvr", dict(p_dmvr=0.9, p_bdof=0.05, p_affine=0, p_bi=0.9, mv_sigma=2.0)),
                                      ("affine", dict(p_dmvr=0, p_bdof=0, p_affine=0.9, p_prof=0.8)),
                                      ("geo", dict(p_geo=0.7, p_dmvr=0.1, p_bdof=0.1))])
def test_mc_modes(b200, oracle, name, kw):
    _compare(b200, oracle, _random_case(name, 11, 416, 240, 10, **kw))


@pytest.mark.parametrize("seed,W,H,bd", [(5, 1920, 1080, 10), (6, 256, 128, 8), (7, 384, 256, 12), (8, 3840, 2160, 10)])
def test_mc_mixed_pictures(b200, oracle, seed, W, H, bd):
    _compare(b200, oracle, _random_case(f"mixed_{seed}", seed, W, H, bd, **({"p_dmvr": 0.0} if bd > 10 else {})))


def test_mc_predict_without_weights(b200, oracle):
    """b200_mc_predict, the entry point without a weights table, on a random mixed picture."""
    case = _random_case("mixed_no_wp", 9, 416, 240, 10)
    a, da = mc_oracle(oracle, case)
    g, pus = case["g"], case["pus"]
    b = mc_dst(g); db = np.zeros_like(da)
    vvdec_b200.check(b200.b200_mc_predict(C.byref(g), abi.plane_ptrs(b), ref_ptrs(case["refs"]), 4, pus.ctypes.data, len(pus), db.ctypes.data, len(db)))
    msg = mc_mismatch(case, a, b, da, db)
    assert msg is None, msg


@pytest.mark.parametrize("seed,W,H,bd", [(21, 416, 240, 10), (22, 256, 128, 8), (23, 1920, 1080, 10)])
def test_mc_explicit_weighted_prediction(b200, oracle, seed, W, H, bd):
    """b200_mc_predict_wp: uni / bi / affine(+PROF) PUs with explicit weights, BCW PUs that bypass them (wpIdx 0)."""
    _compare(b200, oracle, _random_case(f"wp_{seed}", seed, W, H, bd, wp=True, p_dmvr=0.0, p_bdof=0.0, p_affine=0.2, p_bcw=0.3))


@pytest.mark.parametrize("name", list(synth.MC_SWEEP_CASES))
def test_mc_designed_sweep(b200, oracle, name):
    """Every case of the designed sweep: all shapes x tools, every phase pair per tile list, windows on their interior / boundary thresholds at all four
    picture edges, clipMv bounds for CTU 32 / 64 / 128, MVs near +-2^17, affine spread limits, DMVR targets and designed cost surfaces, flat and extreme
    reference content; 8 / 10 / 12 bit, 4:0:0, padded and odd strides (odd: every tile takes the per-sample window path)."""
    _compare(b200, oracle, synth.mc_sweep(name))


def test_mc_sbtmvp_runs(b200, oracle):
    """PU records that are not powers of two: the runs of 8x8 SbTMVP sub-blocks the flattener emits (multiples of 8 up to 128 along the longer side,
    vvdec_glue/flatten_pu.h flattenSbTmvp), uni- and bi-predicted, on the 16-sample tile grid."""
    W, H = 416, 240
    sizes = [(24, 8), (8, 24), (40, 16), (16, 40), (48, 8), (8, 56), (24, 16), (72, 8), (8, 88), (120, 8), (104, 16), (16, 24)]
    pos, used = synth._mc_pack(sizes, W, gap=8)
    assert used <= H
    pus = [synth._mc_tool_pu("bi" if k & 1 else "uni0", x, y, w, h, k) for k, ((w, h), (x, y)) in enumerate(zip(sizes, pos))]
    pus, nd = synth._mc_finish(pus)
    refs = [synth.noise_planes(np.random.default_rng(s), W, H, 10) for s in range(4)]
    _compare(b200, oracle, dict(name="sbtmvp_runs", g=abi.make_geom(W, H, 10), W=W, H=H, bd=10, chroma=1, strides=(W, W // 2, W // 2), pus=pus, ndmvr=nd,
                                refs=refs, tags=["run"] * len(pus), wp=None))


def _refusal_base():
    """A small valid list (256x256 picture, 10 bit): uni, bi, DMVR + BDOF, BDOF, affine, GEO, and a weights table of two entries."""
    W = H = 256
    pus = [synth._mc_pu(0, 0, 16, 16, (0, -1), (5, 3)), synth._mc_pu(16, 0, 16, 16, (0, 2), (5, 3), (-7, 2)),
           synth._mc_pu(32, 0, 16, 16, (0, 2), (16, 0), (-16, 0), synth.PU_DMVR | synth.PU_BDOF), synth._mc_pu(48, 0, 16, 16, (1, 3), (1, 2), (3, 4), synth.PU_BDOF),
           synth._mc_pu(0, 16, 16, 16, (0, 2), (1, 2), (3, 4), synth.PU_AFFINE, cpmv=[[(9, 2), (1, 9)], [(3, 4), (3, 4)]]),
           synth._mc_pu(16, 16, 16, 16, (0, 3), (1, 2), (3, 4), synth.PU_GEO, bcw=17), synth._mc_pu(32, 16, 16, 16, (1, 2), (1, 2), (3, 4))]
    pus, nd = synth._mc_finish(pus)
    ent = np.zeros(2, synth.WP_DTYPE); ent["w0"] = 1; ent["w1"] = 1; ent["shift"] = 1
    return W, H, pus, nd, ent


# one row per refusal: (what, field edits on PU row i or a geometry edit, bit depth)
_PU_REFUSALS = [
    ("slot past numSlots", 0, dict(refSlot=(4, -1))), ("no slot", 0, dict(refSlot=(-1, -1))), ("list-1 slot past numSlots", 1, dict(refSlot=(0, 9))),
    ("width not a multiple of 4", 0, dict(w=6)), ("width 12: a 12-sample tile", 0, dict(w=12)), ("height 28: a 12-sample tile", 0, dict(h=28)), ("height below 4", 0, dict(h=0)), ("width above 128", 0, dict(w=132, x=0)),
    ("off the 4x4 grid", 0, dict(x=2)), ("outside the picture", 6, dict(x=248)), ("below the picture", 6, dict(y=248)),
    ("DMVR entries past numDmvr", 2, dict(dmvrOff=1)), ("DMVR uni-predicted", 2, dict(refSlot=(0, -1))), ("DMVR on 8x8", 2, dict(w=8, h=8)),
    ("DMVR affine", 2, dict(flags=synth.PU_DMVR | synth.PU_AFFINE)), ("BDOF on a small bi PU", 3, dict(w=8, h=8)),
    ("GEO uni-predicted", 5, dict(refSlot=(0, -1))), ("GEO 4 wide", 5, dict(w=4)), ("GEO 128 wide", 5, dict(w=128, h=64, x=0, y=0)),
    ("GEO not a power of two", 5, dict(w=12)), ("GEO with DMVR", 5, dict(flags=synth.PU_GEO | synth.PU_DMVR)), ("GEO with BDOF", 5, dict(flags=synth.PU_GEO | synth.PU_BDOF)),
    ("GEO with affine", 5, dict(flags=synth.PU_GEO | synth.PU_AFFINE)), ("GEO with weights", 5, dict(wpIdx=1)), ("GEO split direction 64", 5, dict(bcwW1=64)),
    ("weights past numWp", 6, dict(wpIdx=3)), ("weights with DMVR", 2, dict(wpIdx=1)), ("weights with BDOF", 3, dict(wpIdx=1)), ("weights with BCW", 6, dict(wpIdx=1, bcwW1=5)),
]
_GEOM_REFUSALS = [("DMVR at 12 bit", dict(bitDepth=12)), ("chromaFormat 2", dict(chromaFormat=2)), ("chromaFormat 3", dict(chromaFormat=3)),
                  ("bit depth 7", dict(bitDepth=7)), ("bit depth 13", dict(bitDepth=13)), ("luma stride below the width", dict(stride=(252, 128, 128))),
                  ("chroma stride below the width", dict(stride=(256, 128, 126)))]


@pytest.mark.parametrize("what,row,edit", _PU_REFUSALS + [(w, None, e) for w, e in _GEOM_REFUSALS], ids=[r[0] for r in _PU_REFUSALS + _GEOM_REFUSALS])
def test_mc_refusals(b200, oracle, what, row, edit):
    """Each rule of the list validation (bucket.cu pu_head) and of the wrapper's geometry checks, alone, makes b200_mc_predict_wp return B200_ERR_PARAM
    and leaves the host destination planes and DMVR deltas as they were."""
    W, H, pus, nd, ent = _refusal_base()
    g = abi.make_geom(W, H, 10)
    rng = np.random.default_rng(3)
    refs = [synth.noise_planes(rng, W, H, 10) for _ in range(4)]
    base = dict(name="refusal_base", g=g, W=W, H=H, bd=10, chroma=1, strides=(W, W // 2, W // 2), pus=pus, ndmvr=nd, refs=refs, tags=["base"] * len(pus), wp=(None, ent))
    _compare(b200, oracle, base)                                                # the unedited list is accepted and right
    if row is None:
        for k, v in edit.items():
            if k == "stride":
                for c in range(3): g.stride[c] = v[c]
            else: setattr(g, k, v)
    else:
        for k, v in edit.items(): pus[k][row] = v
    dst = [np.full((H, W), -7, np.int16), np.full((H // 2, W // 2), -7, np.int16), np.full((H // 2, W // 2), -7, np.int16)]
    dm = np.full((nd + 1, 2), -7, np.int32)
    rc = b200.b200_mc_predict_wp(C.byref(g), abi.plane_ptrs(dst), ref_ptrs(refs), 4, pus.ctypes.data, len(pus), dm.ctypes.data, nd, ent.ctypes.data, len(ent))
    assert rc == -2, (what, rc)
    assert all((p == -7).all() for p in dst) and (dm == -7).all(), what
