#!/usr/bin/env python
"""Generates tests/golden/*.npz from the compiled reference (oracle/_ref/libvvdec_ref.so, i.e. unmodified VVdeC + our shim).
Run where the reference sources have built oracle/_ref:  python tools/make_golden.py
The fixtures hold inputs AND the reference's outputs, so `tests/test_golden_cpu.py` can pin the oracle on machines without oracle/_ref."""
import os, sys, ctypes as C
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vvdec_b200 import abi, synth
from tests import helpers
from tests.helpers import RefTuSyntax, ref_ptrs

ref = helpers.load_ref()
assert ref is not None, "build oracle/_ref first (make -C oracle ref)"
OUT = os.path.join(ROOT, "tests", "golden")
os.makedirs(OUT, exist_ok=True)


def k1():
    rng = np.random.default_rng(101)
    recs, levels, res0, res1, coefs, syn = [], [], [], [], [], []
    fields = [f for f, _ in RefTuSyntax._fields_]
    n = 0
    while n < 160:
        s = RefTuSyntax()
        s.comp = int(rng.choice([0, 0, 1, 2])); s.w = 1 << int(rng.integers(2, 7)); s.h = 1 << int(rng.integers(2, 7))
        cw = s.w >> (1 if s.comp else 0); ch = s.h >> (1 if s.comp else 0)
        if min(cw, ch) < 2: continue
        s.bitDepth = int(rng.choice([8, 10])); s.qp = int(rng.integers(10, 52)); s.predMode = int(rng.integers(0, 2)); s.depQuant = int(rng.integers(0, 2))
        s.intraDirL = int(rng.integers(0, 67)); s.intraDirC = int(rng.choice([0, 1, 18, 50])); s.spsMTS = 1; s.spsIntraMTS = int(rng.integers(0, 2)); s.spsInterMTS = 1
        kind = n % 5
        s.maxScanPosX = min(min(cw, 32), 4 * int(rng.integers(1, 9))) - 1; s.maxScanPosY = min(min(ch, 32), 4 * int(rng.integers(1, 9))) - 1
        if kind == 1 and max(cw, ch) <= 32: s.mtsIdx = 1
        elif kind == 2 and s.comp == 0 and s.predMode == 0 and max(cw, ch) <= 32 and min(cw, ch) >= 4:
            s.mtsIdx = int(rng.integers(2, 6)); s.maxScanPosX = min(s.maxScanPosX, 15); s.maxScanPosY = min(s.maxScanPosY, 15)
        elif kind == 3 and min(cw, ch) >= 4:
            s.predMode = 1; s.spsLFNST = 1; s.lfnstIdx = int(rng.integers(1, 3)); s.sepTree = 1 if s.comp else 0; s.maxScanPosX = s.maxScanPosY = 3; s.spsMTS = 0
        elif kind == 4 and s.comp:
            s.jointCbCr = int(rng.integers(1, 4)); s.jointCbCrSign = int(rng.integers(0, 2))
        lv = np.zeros((ch, cw), np.int16)
        sub = rng.laplace(0, 8, size=(s.maxScanPosY + 1, s.maxScanPosX + 1)).clip(-32768, 32767).astype(np.int16)
        if s.lfnstIdx:
            yy, xx = np.mgrid[0:4, 0:4]; sub[(xx + yy) > 2] = 0
        sub[-1, -1] = sub[-1, -1] or 1
        lv[:s.maxScanPosY + 1, :s.maxScanPosX + 1] = sub
        lvf = lv.reshape(-1).copy()
        r0 = np.zeros(cw * ch, np.int16); r1 = np.zeros(cw * ch, np.int16); rec = abi.Tu(); co = np.zeros(cw * ch + 16, np.int16); nc = C.c_int32(0)
        assert ref.ref_tu_case(C.byref(s), lvf, r0, r1, C.byref(rec), co, C.byref(nc)) == 1
        syn.append([getattr(s, f) for f in fields]); recs.append(np.frombuffer(bytes(rec), np.uint8).copy())
        pad = np.zeros(4096, np.int16)
        for dst, src in ((levels, lvf), (res0, r0), (res1, r1), (coefs, co[:nc.value])):
            p = pad.copy(); p[:len(src)] = src; dst.append(p)
        n += 1
    np.savez_compressed(os.path.join(OUT, "k1_tu_cases.npz"), fields=np.array(fields), syntax=np.array(syn, np.int32), recs=np.array(recs),
                        levels=np.array(levels), res0=np.array(res0), res1=np.array(res1), coefs=np.array(coefs))


def pictures():
    W, H, bd, ctu = 192, 128, 10, 64
    g = abi.make_geom(W, H, bd, ctu=ctu)
    rng = np.random.default_rng(202)
    refs = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
    # K2
    cus = synth.partition(rng, W, H, ctu=ctu)
    pus, nd = synth.gen_pus(rng, cus, W, H, p_affine=0.2, p_prof=1.0)
    out = [np.zeros((H, W), np.int16), np.zeros((H // 2, W // 2), np.int16), np.zeros((H // 2, W // 2), np.int16)]
    dm = np.zeros((nd + 1, 2), np.int32)
    assert ref.ref_mc_predict(0, C.byref(g), abi.plane_ptrs(out), ref_ptrs(refs), pus.ctypes.data, len(pus), dm.ctypes.data, nd) == 0
    np.savez_compressed(os.path.join(OUT, "k2_mc_picture.npz"), geom=[W, H, bd, ctu], pus=pus, ndmvr=nd, dmvr=dm,
                        **{f"ref{s}_{c}": refs[s][c] for s in range(4) for c in range(3)}, **{f"out{c}": out[c] for c in range(3)})
    # K3
    lfV, lfH = synth.gen_lf_grid(rng, cus, W, H, bd)
    sl = np.zeros(2, synth.LFSLICE_DTYPE); sl["beta"] = [[1, -2, 2], [0, 0, 0]]; sl["tc"] = [[-1, 2, 0], [3, -3, 1]]
    cs = np.array([0, 0, 1, 0, 1, 1], np.uint8)
    seq = abi.LfSeq(); seq.ladfEnabled, seq.ladfNumIntervals = 1, 2; seq.ladfQpOffset[0], seq.ladfQpOffset[1] = 1, -2; seq.ladfIntervalLowerBound[1] = 500
    src = refs[0]; o3 = [p.copy() for p in src]
    ref.ref_lf_deblock_picture(0, C.byref(g), abi.plane_ptrs(o3), lfV.ctypes.data, lfH.ctypes.data, cs.ctypes.data, sl.ctypes.data, 2, C.addressof(seq), 3)
    np.savez_compressed(os.path.join(OUT, "k3_deblock_picture.npz"), geom=[W, H, bd, ctu], lfV=lfV, lfH=lfH, slices=sl, ctuSlice=cs,
                        ladf=[1, 2, 1, -2, 0, 500], **{f"in{c}": src[c] for c in range(3)}, **{f"out{c}": o3[c] for c in range(3)})
    # K4
    sao = synth.gen_sao(rng, W, H, ctu, bd, p_on=0.8)
    v = abi.Vb(); v.numVer, v.numHor = 1, 1; v.posX[0], v.posY[0] = 72, 40
    o4 = [np.zeros_like(p) for p in src]
    ref.ref_sao_picture(0, C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(o4), sao.ctypes.data, C.addressof(v))
    np.savez_compressed(os.path.join(OUT, "k4_sao_picture.npz"), geom=[W, H, bd, ctu], sao=sao, vb=[1, 1, 72, 40],
                        **{f"in{c}": src[c] for c in range(3)}, **{f"out{c}": o4[c] for c in range(3)})
    # K5
    t = synth.gen_alf(rng, W, H, ctu, bd, n_aps=2)
    T = abi.make_alf_tables(t)
    o5 = [np.zeros_like(p) for p in src]
    ref.ref_alf_picture(0, C.byref(g), abi.plane_ptrs(src), abi.plane_ptrs(o5), t["ctus"].ctypes.data, C.byref(T))
    np.savez_compressed(os.path.join(OUT, "k5_alf_picture.npz"), geom=[W, H, bd, ctu], ctus=t["ctus"], lumaCoeff=t["lumaCoeff"][16:], lumaClip=t["lumaClip"][16:],
                        chromaCoeff=t["chromaCoeff"], chromaClip=t["chromaClip"], cc0=t["cc"][0], cc1=t["cc"][1],
                        **{f"in{c}": src[c] for c in range(3)}, **{f"out{c}": o5[c] for c in range(3)})


def chain():
    """Whole back end on one small picture with the tools added after the first fixtures: GEO, explicit weighted prediction, LMCS with
    chroma scaling, on top of K2 -> K1 -> K3 -> K4 -> K5; output of the reference arm (the reference's own kernels, SIMD off)."""
    W, H, bd, ctu = 256, 128, 10, 128
    g = abi.make_geom(W, H, bd, ctu=ctu)
    rng = np.random.default_rng(303)
    refs = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
    pic = synth.gen_picture(rng, W, H, bd, ctu=ctu, dst_slot=0, wp=True, lmcs=True, pu_kw=dict(p_dmvr=0.0, p_bdof=0.0, p_bcw=0.3, p_geo=0.2), tu_kw=dict(p_cbf=0.7))
    vp = pic["lmcs"]["vpdus"]                                   # the reference arm's CU structure is one CU per CTU (tests/test_lmcs_oracle_vs_ref.py)
    for j in range((H + 63) // 64):
        for i in range((W + 63) // 64):
            cx, cy = i * 64 // ctu * ctu, j * 64 // ctu * ctu
            vp[j * ((W + 63) // 64) + i] = (cx, cy, cx > 0, cy > 0)
    out = [np.zeros((H, W), np.int16), np.zeros((H // 2, W // 2), np.int16), np.zeros((H // 2, W // 2), np.int16)]
    ref.ref_set_wp(pic["wpRaw"].ctypes.data)
    try: ref.ref_decompress_picture_out(C.byref(g), ref_ptrs(refs), C.byref(pic["struct"]), 2, 0, abi.plane_ptrs(out))
    finally: ref.ref_set_wp(None)
    np.savez_compressed(os.path.join(OUT, "chain_geo_wp_lmcs_picture.npz"), geom=[W, H, bd, ctu], **synth.save_picture(pic),
                        **{f"ref{s}_{c}": refs[s][c] for s in range(4) for c in range(3)}, **{f"out{c}": out[c] for c in range(3)})


def film_grain():
    """Film grain: an FGC SEI (frequency-filtering model, three components) through the reference's firmware (FilmGrain::updateFGC) and its SIMD
    line kernels on the third frame of a sequence (seed state carried over); tables as the glue flattener exports them."""
    W, H, bd = 208, 96, 10
    rng = np.random.default_rng(404)
    sei = synth.gen_fgc_sei(rng, 0, (1, 1, 1), max_scale=128)
    src = synth.noise_planes(rng, W, H, bd)
    out = [p.copy() for p in src]
    pattern = np.zeros((2, 8, 64, 64), np.int8); sLUT = np.zeros((3, 256), np.uint8); pLUT = np.zeros((3, 256), np.uint8)
    seeds = np.zeros((H + 15) // 16, np.uint32); shift = C.c_int(0); present = np.zeros(3, np.uint8)
    strides = (C.c_ssize_t * 3)(*[p.shape[1] for p in out])
    assert ref.ref_film_grain(sei.ctypes.data, 0, bd, W, H, 3, abi.plane_ptrs(out), strides, pattern.ctypes.data, sLUT.ctypes.data, pLUT.ctypes.data,
                              seeds.ctypes.data, C.byref(shift), present.ctypes.data) == 0
    np.savez_compressed(os.path.join(OUT, "film_grain_fgc.npz"), geom=[W, H, bd], sei=sei, pattern=pattern, sLUT=sLUT, pLUT=pLUT, seeds=seeds, shift=shift.value,
                        present=present, **{f"src{c}": src[c] for c in range(3)}, **{f"out{c}": out[c] for c in range(3)})


def intra():
    """An all-intra picture through the reference's IntraPrediction (SIMD kernels): every CU predicted from the reconstruction of the earlier ones
    (regular modes, MRL, BDPCM prediction), pred + residual on about half of the CUs; records from the glue flattener."""
    rng = np.random.default_rng(505)
    g, planes, resi, recs, out = helpers.intra_picture_case(ref, rng, 192, 128, 10, 64, 1, min_size=8)
    np.savez_compressed(os.path.join(OUT, "k6_intra_picture.npz"), geom=[192, 128, 10, 64], recs=recs, **{f"src{c}": planes[c] for c in range(3)},
                        **{f"resi{c}": resi[c] for c in range(3)}, **{f"out{c}": out[c] for c in range(3)})


def lmcs():
    """LMCS sweep pictures (synth.lmcs_sweep: designed VPDU neighbour averages on every pivot of full_bins, DC / 4-sample / joint-CbCr chroma TUs) at 8
    and 12 bit through the reference arm (its own calculateChromaAdjVpduNei / scaleSignal / applyLut, SIMD off).  The sweep's records are CTU origins at
    CTU 32, the reference arm's one CU per CTU.  The inputs are rebuilt from the sweep; the fixture keeps the `given` luma as a check of that."""
    names = ["vpdu_full_bins_8bit_ctu32", "vpdu_full_bins_12bit_ctu32"]
    out = dict(names=np.array(names))
    for name in names:
        c = synth.lmcs_sweep(name)
        o = [np.zeros((c["H"], c["W"]), np.int16), np.zeros((c["H"] // 2, c["W"] // 2), np.int16), np.zeros((c["H"] // 2, c["W"] // 2), np.int16)]
        ref.ref_decompress_picture_out(C.byref(c["g"]), ref_ptrs(c["dpb"]), C.byref(c["pic"]["struct"]), 2, 0, abi.plane_ptrs(o))
        out[f"{name}_given0"] = c["pic"]["given"][0]
        out.update({f"{name}_out{k}": o[k] for k in range(3)})
    np.savez_compressed(os.path.join(OUT, "lmcs_pictures.npz"), **out)


LF_DERIVE_CASES = [("B_mixed", 1, (416, 240)), ("B_affine_heavy", 2, (416, 240)), ("I_picture", 1, (416, 240)), ("P_picture", 2, (416, 240)), ("B_isp", 3, (416, 240)),
                   ("B_5slices_no_lf_across_ctu64", 1, (416, 240)), ("I_6slices_no_lf_across_ctu64", 2, (416, 240)), ("B_local_dual_tree_isp", 1, (416, 240)),
                   ("I_local_dual_tree", 3, (416, 240)), ("B_ctu32_8bit", 1, (200, 136)), ("B_mixed", 2, (200, 136)), ("B_3slices", 3, (416, 240))]


def lf_derive():
    """Seam pictures (tests/test_lf_derive_cpu.py CASES) as the drop-in class flattens them with the device edge derivation switched on — CU / TU / PU records,
    CTU ranges, slice tables — and the reference's own edge grids of the same pictures (calcFilterStrengthsCTU + flattenLfCtu)."""
    from tests.test_lf_derive_cpu import CASES, flatten_grids, records_of
    out = dict(names=np.array([f"{n}-s{s}-{w}x{h}" for n, s, (w, h) in LF_DERIVE_CASES]))
    for k, (name, seed, (w, h)) in enumerate(LF_DERIVE_CASES):
        case = helpers.SeamCase(ref, np.random.default_rng(seed), w, h, **CASES[name])
        wantV, wantH, _ = flatten_grids(case, False)
        _, _, flat = flatten_grids(case, True)
        r = records_of(flat, case.g)
        g = case.g
        out[f"{k}_geom"] = np.array([g.width, g.height, g.chromaFormat, g.bitDepth, g.ctuSize], np.int32)
        out.update({f"{k}_{f}": v for f, v in r.items()})
        out[f"{k}_lfV"] = wantV; out[f"{k}_lfH"] = wantH
    np.savez_compressed(os.path.join(OUT, "lf_derive_pictures.npz"), **out)


if __name__ == "__main__":
    import sys
    if len(sys.argv) > 1: [globals()[n]() for n in sys.argv[1:]]
    else: k1(); pictures(); chain(); film_grain(); intra(); lmcs(); lf_derive()
    print({f: os.path.getsize(os.path.join(OUT, f)) for f in sorted(os.listdir(OUT))})
