"""Oracle vs the committed golden vectors (tests/golden/*.npz, generated from the compiled reference by tools/make_golden.py).
These run without oracle/_ref and without a GPU; the same fixtures are replayed on the GPU by tests/test_golden_gpu.py."""
import os, ctypes as C
import numpy as np
import pytest
from vvdec_b200 import abi, synth

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    return np.load(os.path.join(G, name))


def _planes(z, prefix):
    return [np.ascontiguousarray(z[f"{prefix}{c}"]) for c in range(3)]


def run_k1(fn_residual):
    z = _load("k1_tu_cases.npz")
    fields = list(z["fields"])
    for i in range(len(z["syntax"])):
        s = dict(zip(fields, z["syntax"][i]))
        rec = abi.Tu.from_buffer_copy(z["recs"][i].tobytes())
        cw, ch = 1 << rec.log2w, 1 << rec.log2h
        planes = [np.zeros((128, 128), np.int16), np.zeros((64, 64), np.int16), np.zeros((64, 64), np.int16)]
        fn_residual(abi.make_geom(128, 128, int(s["bitDepth"])), planes, (abi.Tu * 1)(rec), np.ascontiguousarray(z["coefs"][i]))
        assert np.array_equal(planes[rec.comp][:ch, :cw].reshape(-1), z["res0"][i][:cw * ch]), (i, s)
        if rec.ict:
            assert np.array_equal(planes[2 if rec.comp == 1 else 1][:ch, :cw].reshape(-1), z["res1"][i][:cw * ch]), (i, s)


def test_k1_golden(oracle):
    run_k1(lambda g, planes, recs, coefs: oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(planes), recs, 1, coefs, None, 1))


def geom_of(z):
    W, H, bd, ctu = [int(v) for v in z["geom"]]
    return abi.make_geom(W, H, bd, ctu=ctu), W, H


def run_k2(fn):
    z = _load("k2_mc_picture.npz"); g, W, H = geom_of(z)
    refs = [[np.ascontiguousarray(z[f"ref{s}_{c}"]) for c in range(3)] for s in range(4)]
    pus = np.ascontiguousarray(z["pus"]); nd = int(z["ndmvr"])
    out = [np.zeros((H, W), np.int16), np.zeros((H // 2, W // 2), np.int16), np.zeros((H // 2, W // 2), np.int16)]
    dm = np.zeros((nd + 1, 2), np.int32)
    fn(g, out, refs, pus, dm)
    for c in range(3): assert np.array_equal(out[c], z[f"out{c}"]), f"plane {c}"
    assert np.array_equal(dm, z["dmvr"])


def test_k2_golden(oracle):
    from tests.helpers import ref_ptrs
    run_k2(lambda g, out, refs, pus, dm: oracle.orc_mc_predict(C.byref(g), abi.plane_ptrs(out), ref_ptrs(refs), pus.ctypes.data, len(pus), dm.ctypes.data))


def k3_inputs():
    z = _load("k3_deblock_picture.npz"); g, W, H = geom_of(z)
    seq = abi.LfSeq(); l = [int(v) for v in z["ladf"]]
    seq.ladfEnabled, seq.ladfNumIntervals = l[0], l[1]; seq.ladfQpOffset[0], seq.ladfQpOffset[1] = l[2], l[3]; seq.ladfIntervalLowerBound[0], seq.ladfIntervalLowerBound[1] = l[4], l[5]
    return z, g, _planes(z, "in"), np.ascontiguousarray(z["lfV"]), np.ascontiguousarray(z["lfH"]), np.ascontiguousarray(z["ctuSlice"]), np.ascontiguousarray(z["slices"]), seq


def test_k3_golden(oracle):
    z, g, p, lfV, lfH, cs, sl, seq = k3_inputs()
    oracle.orc_lf_deblock(C.byref(g), abi.plane_ptrs(p), lfV.ctypes.data, lfH.ctypes.data, cs.ctypes.data, sl.ctypes.data, C.addressof(seq), 3)
    for c in range(3): assert np.array_equal(p[c], z[f"out{c}"])


def k4_inputs():
    z = _load("k4_sao_picture.npz"); g, W, H = geom_of(z)
    v = abi.Vb(); v.numVer, v.numHor, v.posX[0], v.posY[0] = [int(x) for x in z["vb"]]
    return z, g, _planes(z, "in"), np.ascontiguousarray(z["sao"]), v


def test_k4_golden(oracle):
    z, g, src, sao, v = k4_inputs()
    out = [np.zeros_like(p) for p in src]
    oracle.orc_sao_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(out), sao.ctypes.data, C.addressof(v))
    for c in range(3): assert np.array_equal(out[c], z[f"out{c}"])


def k5_inputs():
    z = _load("k5_alf_picture.npz"); g, W, H = geom_of(z)
    fixed = synth._fixed_sets()
    coef = np.ascontiguousarray(np.concatenate([fixed, z["lumaCoeff"]]).astype(np.int16))
    clip = np.ascontiguousarray(np.concatenate([np.full_like(fixed, 1 << int(z["geom"][2])), z["lumaClip"]]).astype(np.int16))
    t = dict(lumaCoeff=coef, lumaClip=clip, chromaCoeff=np.ascontiguousarray(z["chromaCoeff"]), chromaClip=np.ascontiguousarray(z["chromaClip"]),
             cc=[np.ascontiguousarray(z["cc0"]), np.ascontiguousarray(z["cc1"])], ctus=np.ascontiguousarray(z["ctus"]))
    return z, g, _planes(z, "in"), t, abi.make_alf_tables(t)


def test_k5_golden(oracle):
    z, g, src, t, T = k5_inputs()
    out = [np.zeros_like(p) for p in src]
    oracle.orc_alf_picture(C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(out), t["ctus"].ctypes.data, C.byref(T))
    for c in range(3): assert np.array_equal(out[c], z[f"out{c}"])


def chain_inputs():
    z = _load("chain_geo_wp_lmcs_picture.npz"); g, W, H = geom_of(z)
    refs = [[np.ascontiguousarray(z[f"ref{s}_{c}"]) for c in range(3)] for s in range(4)]
    from vvdec_b200 import synth
    pic = synth.load_picture(z, g.bitDepth)
    return z, g, refs, pic


def test_chain_golden(oracle):
    """Whole chain with GEO + explicit weighted prediction + LMCS (chroma scaling) against the reference arm's stored output."""
    from tests.helpers import oracle_decompress
    z, g, refs, pic = chain_inputs()
    assert (pic["pus"]["flags"] & 128).any() and (pic["pus"]["wpIdx"] != 0).any()
    out, _ = oracle_decompress(oracle, g, refs, pic)
    for c in range(3): assert np.array_equal(out[c], z[f"out{c}"]), f"plane {c}"


def test_lmcs_golden(oracle):
    """tests/golden/lmcs_pictures.npz: LMCS sweep pictures at 8 and 12 bit (designed VPDU neighbourhoods, scaled chroma TUs) through the reference arm."""
    from tests.helpers import oracle_decompress
    z = _load("lmcs_pictures.npz")
    assert len(z["names"]) == 2
    for name in [str(n) for n in z["names"]]:
        c = synth.lmcs_sweep(name)
        assert np.array_equal(c["pic"]["given"][0], z[f"{name}_given0"]), name     # the sweep still builds the fixture's input
        out, _ = oracle_decompress(oracle, c["g"], c["dpb"], c["pic"])
        for k in range(3): assert np.array_equal(out[k], z[f"{name}_out{k}"]), (name, k)


def test_film_grain_golden(oracle):
    """tests/golden/film_grain_fgc.npz: tables from the reference's FGC firmware, output of its SIMD line kernels (third frame of a sequence)."""
    z = _load("film_grain_fgc.npz")
    W, H, bd = [int(v) for v in z["geom"]]
    got = _planes(z, "src")
    strides = (C.c_ssize_t * 3)(*[p.shape[1] for p in got])
    tabs = [np.ascontiguousarray(z[k]) for k in ("pattern", "sLUT", "pLUT", "seeds", "present")]
    oracle.orc_film_grain(abi.plane_ptrs(got), strides, W, H, bd, tabs[0].ctypes.data, tabs[1].ctypes.data, tabs[2].ctypes.data, tabs[3].ctypes.data, int(z["shift"]), tabs[4].ctypes.data)
    for c in range(3):
        assert np.array_equal(got[c], z[f"out{c}"]), c


def test_k6_intra_golden(oracle):
    """tests/golden/k6_intra_picture.npz: an all-intra picture chained through the reference's IntraPrediction (SIMD), with residual adds."""
    z = _load("k6_intra_picture.npz")
    W, H, bd, ctu = [int(v) for v in z["geom"]]
    g = abi.make_geom(W, H, bd, ctu=ctu)
    got, resi = _planes(z, "src"), _planes(z, "resi")
    recs = np.ascontiguousarray(z["recs"])
    oracle.orc_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), recs.ctypes.data, len(recs))
    for c in range(3):
        assert np.array_equal(got[c], z[f"out{c}"]), c
