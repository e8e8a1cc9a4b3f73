"""Filter flatteners (vvdec_b200/vvdec_glue/flatten_filters.h): the reference's CtuData / APS / LoopFilterParam structures are filled from a
synthetic picture (the same way the filter shims feed the real LoopFilter / SAO / ALF), then flattened again by the glue — the result must be
the input, with the SAO availability coming from the real deriveLoopFilterBoundaryAvailibility."""
import ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth

pytestmark = pytest.mark.ref


@pytest.mark.parametrize("W,H,ctu", [(416, 240, 128), (384, 256, 64), (200, 136, 32)])
def test_filter_flatteners_round_trip(ref, W, H, ctu):
    rng = np.random.default_rng(W)
    bd = 10
    g = abi.make_geom(W, H, bd, ctu=ctu)
    pic = synth.gen_picture(rng, W, H, bd, ctu=ctu)
    lfV, lfH, sao, alf = pic["lfV"], pic["lfH"], pic["sao"], pic["alf"]
    T = pic["alfTabs"]
    lfVo, lfHo = np.zeros_like(lfV), np.zeros_like(lfH)
    saoO, alfO = np.zeros_like(sao), np.zeros_like(alf["ctus"])
    outs = [np.zeros_like(alf[k]) for k in ("lumaCoeff", "lumaClip", "chromaCoeff", "chromaClip")] + [np.zeros_like(alf["cc"][0]), np.zeros_like(alf["cc"][1])]
    counts = (C.c_int32 * 4)()
    V = C.c_void_p
    ref.ref_flatten_filters.argtypes = [C.POINTER(abi.Geom)] + [V] * 4 + [C.POINTER(abi.AlfTables)] + [V] * 10 + [C.POINTER(C.c_int32)]
    rc = ref.ref_flatten_filters(C.byref(g), lfV.ctypes.data, lfH.ctypes.data, sao.ctypes.data, alf["ctus"].ctypes.data, C.byref(T),
                                 lfVo.ctypes.data, lfHo.ctypes.data, saoO.ctypes.data, alfO.ctypes.data, *[o.ctypes.data for o in outs], counts)
    assert rc == 0
    assert np.array_equal(lfV.view(np.uint8), lfVo.view(np.uint8)) and np.array_equal(lfH.view(np.uint8), lfHo.view(np.uint8))
    # the picture path runs these grids unchecked: they must meet the rule b200_lf_deblock enforces
    assert synth.lf_grid_problems(lfVo, 0, g) == [] and synth.lf_grid_problems(lfHo, 1, g) == []
    assert np.array_equal(alf["ctus"].view(np.uint8), alfO.view(np.uint8))
    assert list(counts) == [alf["lumaCoeff"].shape[0], alf["chromaCoeff"].shape[0], alf["cc"][0].shape[0], alf["cc"][1].shape[0]]
    for k, o in zip(("lumaCoeff", "lumaClip", "chromaCoeff", "chromaClip"), outs): assert np.array_equal(alf[k], o), k
    assert np.array_equal(alf["cc"][0], outs[4]) and np.array_equal(alf["cc"][1], outs[5])
    # SAO: type / band / the offsets the filter reads / availability (one slice, one tile: picture boundaries only)
    assert np.array_equal(sao["type"], saoO["type"]) and np.array_equal(sao["avail"], saoO["avail"])
    for c in range(3):
        bo = sao["type"][:, c] == 4; eo = sao["type"][:, c] < 4
        assert np.array_equal(sao["band"][bo, c], saoO["band"][bo, c])
        assert np.array_equal(sao["offset"][bo, c, :4], saoO["offset"][bo, c, :4]) and np.array_equal(sao["offset"][eo, c], saoO["offset"][eo, c])


@pytest.mark.parametrize("seed,kw", [(1, dict()), (2, dict(ctu=32, bd=8)), (3, dict(ctu=64, slice_type=2, isp=30)), (4, dict(affine=60, split=85)),
                                     (5, dict(tools=None, slices=3, ctu=32)),
                                     (6, dict(slices=3, lf_across_slices=False))])
def test_flattened_deblocking_grids_are_legal(ref, seed, kw):
    """The grids the glue flattens from the reference's own calcFilterStrengths (sub-block lengths 5 and 2 of affine / SbTMVP CUs, 4-wide CUs, CTU 32
    rows, intra pictures) meet the rule of the flat pass: the picture path runs them without checking.  Its SAO / ALF records, clip and pad flags of
    slices that do not filter across each other included, meet the rule of b200_sao_picture / b200_alf_picture."""
    from tests import helpers
    case = helpers.SeamCase(ref, np.random.default_rng(seed), 416, 240, **kw)
    pic, rc = case.flatten()
    assert pic is not None, rc
    W4, H4 = case.W // 4, case.H // 4
    lfV, lfH = pic["lfV"].reshape(H4, W4), pic["lfH"].reshape(H4, W4)
    assert synth.lf_grid_problems(lfV, 0, case.g) == [] and synth.lf_grid_problems(lfH, 1, case.g) == []
    # the SAO / ALF records the glue flattens meet the rule b200_sao_picture / b200_alf_picture enforce, which the picture path shares
    st = pic["struct"]
    if st.flags & abi.PIC_SAO: assert synth.k45_record_problems("sao", case.g, pic["sao"]) == []
    if st.flags & abi.PIC_ALF:
        T = pic["alfTabs"]
        t = dict(lumaCoeff=pic["alfArrays"]["lumaCoeff"].reshape(-1, 4, 25, 13), chromaCoeff=np.zeros((T.numChromaAlts, 7)), cc=[np.zeros((T.numCc[c], 7)) for c in range(2)])
        assert synth.k45_record_problems("alf", case.g, pic["alf"]["ctus"], t) == []
    lens = {int(v) >> 4 & 7 for v in lfV["len"][lfV["bs"] & 3 > 0]} | {int(v) & 7 for v in lfV["len"][lfV["bs"] & 3 > 0]}
    assert lens >= {1, 3}, lens
