"""LMCS on the device at 8, 10 and 12 bit: the designed sweep (synth.lmcs_sweep) through b200_decompress_picture, bit-exact against the C oracle chain
(helpers.oracle_decompress) and, for two pictures, against the reference arm's output stored in tests/golden/lmcs_pictures.npz.  Covers the inverse map
(both kernel paths), the forward map in K2's luma stores, the per-VPDU chroma scale and its use in K1, the clip16 bound, 4:0:0, models that change
between pictures, and the refusal of LMCS models and VPDU records the kernels cannot read safely."""
import ctypes as C
import os
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth
from tests.helpers import oracle_decompress

pytestmark = pytest.mark.gpu
BDS = (8, 10, 12)
SLOT = 4


class Ctx:
    def __init__(self, b200, case, arenas=2):
        self.b200, self.case = b200, case
        self.h = C.c_void_p()
        vvdec_b200.check(b200.b200_ctx_create(C.byref(self.h), C.byref(case["g"]), 6, arenas, -1))
        for s, pl in enumerate(case["dpb"]): vvdec_b200.check(b200.b200_ctx_load_slot(self.h, s, abi.plane_ptrs(pl)))

    def frame(self, want):
        got = [np.full_like(p, -9) for p in want]
        vvdec_b200.check(self.b200.b200_get_frame(self.h, SLOT, abi.plane_ptrs(got)))
        return got

    def decode(self, pic, want):
        a = self.b200.b200_decompress_picture(self.h, C.byref(pic["struct"]))
        assert a >= 0, self.b200.b200_last_error()
        vvdec_b200.check(self.b200.b200_wait_picture(self.h, a, None, 0))
        return self.frame(want)

    def close(self):
        self.b200.b200_ctx_destroy(self.h)


def planes_of(case):
    return 3 if case["chroma"] else 1


def mismatch(case, got, want, what=""):
    for c in range(planes_of(case)):
        bad = np.argwhere(got[c] != want[c])
        if len(bad):
            y, x = (int(v) for v in bad[0])
            return f"{case['name']}{what}: plane {c}: {len(bad)} samples differ, first at (y={y}, x={x}): {got[c][y, x]} vs {want[c][y, x]}"
    return None


def run_case(b200, oracle, case):
    want, _ = oracle_decompress(oracle, case["g"], case["dpb"], case["pic"])
    ctx = Ctx(b200, case)
    try: got = ctx.decode(case["pic"], want)
    finally: ctx.close()
    assert mismatch(case, got, want) is None, mismatch(case, got, want)
    return got, want


@pytest.mark.parametrize("stride", ["stride8", "odd"])
@pytest.mark.parametrize("bd", BDS)
def test_inverse_map(b200, oracle, bd, stride):
    """3a: a ramp of every value as `given` luma, no PUs / TUs, filters off: the output luma is invLUT[v] for every model, through the 16-byte path
    (stride a multiple of 8) and the per-sample path (odd stride).  The models follow each other in one context."""
    first = synth.lmcs_sweep(f"inverse_{synth.LMCS_MODELS[0]}_{bd}bit_{stride}")
    ctx = Ctx(b200, first)
    try:
        for m in synth.LMCS_MODELS:
            case = synth.lmcs_sweep(f"inverse_{m}_{bd}bit_{stride}")
            want, _ = oracle_decompress(oracle, case["g"], case["dpb"], case["pic"])
            W = case["W"]; lut = case["pic"]["lmcs"]["invLUT"]
            assert np.array_equal(want[0][:, :W], lut[case["pic"]["given"][0][:, :W]])
            got = ctx.decode(case["pic"], want)
            assert mismatch(case, got, want) is None, mismatch(case, got, want)
    finally:
        ctx.close()


@pytest.mark.parametrize("model", ["compress", "expand_max"])
@pytest.mark.parametrize("bd", BDS)
def test_forward_map(b200, oracle, bd, model):
    """3b: zero-MV uni PUs of several sizes and one bi PU with both references in the slot that holds the ramp: the luma after the inverse map is
    invLUT[fwd(v)] (compress: invLUT is injective on the forward range, so a wrong forward value shows; expand_max: slopes near 8x)."""
    case = synth.lmcs_sweep(f"forward_{model}_{bd}bit")
    got, want = run_case(b200, oracle, case)
    m = case["pic"]["lmcs"]
    f = np.clip(synth.lmcs_fwd(m, case["dpb"][0][0]), 0, (1 << bd) - 1)
    assert np.array_equal(got[0], m["invLUT"][f])


@pytest.mark.parametrize("var", ["ctu32", "ctu64", "ctu128"])
@pytest.mark.parametrize("bd", BDS)
def test_vpdu_chroma_scale(b200, oracle, bd, var):
    """3c: designed neighbour averages on every pivot of the model (CTU 32 / 64), CUs over several VPDUs and walks clamped at the picture's last row /
    column (CTU 128 at 232x120, CTU 64 at 200x136); a DC chroma TU per VPDU shows its scale, 4-sample TUs stay unscaled, joint CbCr is scaled."""
    name = [n for n in synth.LMCS_SWEEP if n.startswith("vpdu_") and n.endswith(f"_{bd}bit_{var}")][0]
    run_case(b200, oracle, synth.lmcs_sweep(name))


def test_scaling_extremes(b200, oracle):
    """3d: crs_min at 12 bit, chroma scale 16384 and residuals of +-2^bd: the scaled residual reaches -32768 (clip16)."""
    got, want = run_case(b200, oracle, synth.lmcs_sweep("extremes_crs_min_12bit"))
    assert (got[1] == 0).any() and (got[1] == 4095).any()


@pytest.mark.parametrize("adj", ["adj", "noadj"])
@pytest.mark.parametrize("bd", BDS)
def test_yuv400(b200, oracle, bd, adj):
    """3e: 4:0:0 with LMCS, chroma scaling flag on and off: forward map in K2, luma TUs, inverse map."""
    run_case(b200, oracle, synth.lmcs_sweep(f"yuv400_fine_pivots_{bd}bit_{adj}"))


def with_model(case, name):
    """The case's picture under another designed model (same VPDU records)."""
    m = synth.lmcs_model(name, case["bd"], vpdus=case["pic"]["lmcs"]["vpdus"])
    pic = dict(case["pic"], lmcs=m)
    st = abi.Picture.from_buffer_copy(case["pic"]["struct"]); st.lmcs = C.addressof(m["struct"]); pic["struct"] = st
    return pic


@pytest.mark.parametrize("bd", BDS)
def test_models_change_between_pictures(b200, oracle, bd):
    """3f: three pictures with different models over two arenas (the third reuses the first arena), then both arenas run again: each run matches its
    own picture's model, so no LMCS table of an earlier picture survives in an arena."""
    case = synth.lmcs_sweep(f"vpdu_full_bins_{bd}bit_ctu32")
    pics = [case["pic"], with_model(case, "crs_min"), with_model(case, "expand_max")]
    wants = [oracle_decompress(oracle, case["g"], case["dpb"], p)[0] for p in pics]
    assert not np.array_equal(wants[0][1], wants[1][1]) and not np.array_equal(wants[0][0], wants[2][0])
    ctx = Ctx(b200, case)
    try:
        arena = []
        for i, p in enumerate(pics):
            a = b200.b200_pic_upload(ctx.h, C.byref(p["struct"])); assert a >= 0, b200.b200_last_error()
            vvdec_b200.check(b200.b200_pic_run(ctx.h, a)); vvdec_b200.check(b200.b200_wait_picture(ctx.h, a, None, 0))
            assert mismatch(case, ctx.frame(wants[i]), wants[i], f" picture {i}") is None
            arena.append(a)
        assert arena[2] == arena[0] != arena[1]
        for a, i in ((arena[1], 1), (arena[0], 2)):                     # re-run what each arena holds now
            vvdec_b200.check(b200.b200_pic_run(ctx.h, a)); vvdec_b200.check(b200.b200_wait_picture(ctx.h, a, None, 0))
            assert mismatch(case, ctx.frame(wants[i]), wants[i], f" re-run of picture {i}") is None
    finally:
        ctx.close()


def test_golden_fixture(b200, oracle):
    """tests/golden/lmcs_pictures.npz: the reference arm's output (SIMD off) for an 8-bit and a 12-bit VPDU sweep picture, through the device."""
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lmcs_pictures.npz"))
    for name in [str(n) for n in z["names"]]:
        case = synth.lmcs_sweep(name)
        assert np.array_equal(case["pic"]["given"][0], z[f"{name}_given0"])
        got, want = run_case(b200, oracle, case)
        for c in range(3): assert np.array_equal(got[c], z[f"{name}_out{c}"]), (name, c)


# ---- 4: refusals.  Each mutation breaks one rule of rules.cuh; the picture is refused with the rule's message before any kernel reads it, and the
# same context then decodes the unchanged picture.
def _model_bad(field, bd):
    org = (1 << bd) // 16
    def f(L):
        if field == "minBin_negative": L.minBinIdx = -1
        elif field == "maxBin_16": L.maxBinIdx = 16
        elif field == "minBin_above_maxBin": L.minBinIdx, L.maxBinIdx = 9, 8
        elif field == "pivot0": L.reshapePivot[0] = 1
        elif field == "pivot_decreasing": L.reshapePivot[8] = L.reshapePivot[9] + 1
        elif field == "pivot16_above": L.reshapePivot[16] = (1 << bd) + 1
        elif field == "inputPivot": L.inputPivot[5] = 5 * org + 1
        elif field == "orgCW": L.orgCW = org * 2
    return f


MODEL_RULES = {"minBin_negative": b"bins", "maxBin_16": b"bins", "minBin_above_maxBin": b"bins", "pivot0": b"reshapePivot[0]",
               "pivot_decreasing": b"decreases", "pivot16_above": b"above 2^bitDepth", "inputPivot": b"inputPivot", "orgCW": b"orgCW"}


def test_refuses_bad_models(b200, oracle):
    for bd in BDS:
        case = synth.lmcs_sweep(f"vpdu_full_bins_{bd}bit_ctu32")
        want, _ = oracle_decompress(oracle, case["g"], case["dpb"], case["pic"])
        ctx = Ctx(b200, case)
        try:
            for rule, msg in MODEL_RULES.items():
                L = case["pic"]["lmcs"]["struct"]
                saved = abi.Lmcs.from_buffer_copy(L)
                _model_bad(rule, bd)(L)
                try:
                    assert b200.b200_decompress_picture(ctx.h, C.byref(case["pic"]["struct"])) == -2, (bd, rule)
                    err = b200.b200_last_error()
                    assert b"b200_pic_upload: LMCS model" in err and msg in err, (bd, rule, err)
                finally:
                    C.memmove(C.byref(L), C.byref(saved), C.sizeof(abi.Lmcs))
                got = ctx.decode(case["pic"], want)
                assert mismatch(case, got, want, f" after {rule}") is None
        finally:
            ctx.close()


def _vpdu_bad(rule, case):
    """(record index, new field values) breaking one VPDU rule; CTU 32, 256x384: VPDU = CTU, raster of 8 per row."""
    W, H = case["W"], case["H"]
    return {"x_outside": (9, dict(x=W)), "y_outside": (9, dict(y=H)), "left_at_x0": (8, dict(availLeft=1)), "above_at_y0": (1, dict(availAbove=1)),
            "origin_right_of_vpdu": (9, dict(x=40)), "origin_below_vpdu": (9, dict(y=40)), "origin_in_ctu_to_the_left": (9, dict(x=0, availLeft=0)),
            "origin_in_ctu_above": (9, dict(y=0, availAbove=0))}[rule]


VPDU_RULES = ("x_outside", "y_outside", "left_at_x0", "above_at_y0", "origin_right_of_vpdu", "origin_below_vpdu", "origin_in_ctu_to_the_left", "origin_in_ctu_above")


def test_refuses_bad_vpdu_records(b200, oracle):
    case = synth.lmcs_sweep("vpdu_full_bins_10bit_ctu32")
    vp = case["pic"]["lmcs"]["vpdus"]
    assert (int(vp[9]["x"]), int(vp[9]["y"])) == (32, 32) and (int(vp[8]["x"]), int(vp[1]["y"])) == (0, 0)
    want, _ = oracle_decompress(oracle, case["g"], case["dpb"], case["pic"])
    ctx = Ctx(b200, case)
    try:
        for rule in VPDU_RULES:
            i, fields = _vpdu_bad(rule, case)
            saved = vp[i].copy()
            for k, v in fields.items(): vp[i][k] = v
            try:
                assert b200.b200_decompress_picture(ctx.h, C.byref(case["pic"]["struct"])) == -2, rule
                err = b200.b200_last_error()
                assert b"b200_pic_run: an LMCS VPDU record is invalid" in err, (rule, err)
            finally:
                vp[i] = saved
            got = ctx.decode(case["pic"], want)
            assert mismatch(case, got, want, f" after {rule}") is None
    finally:
        ctx.close()
