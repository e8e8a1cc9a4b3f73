"""Picture-level parity on the GPU: b200_decompress_picture (DecLibRecon seam, device-resident DPB, all five kernel families
chained) vs the pinned oracle chain, over a short GOP where later pictures reference earlier reconstructed ones."""
import ctypes as C
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth
from tests.helpers import oracle_decompress, intra_kernel, cclm_refusal_rows

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed,W,H,flagsets", [(1, 416, 240, [(1, 1, 1), (1, 0, 1), (0, 0, 0), (1, 1, 0)]), (2, 1920, 1080, [(1, 1, 1), (1, 1, 1)])])
def test_gop_decompress(b200, oracle, seed, W, H, flagsets):
    rng = np.random.default_rng(seed)
    bd = 10
    g = abi.make_geom(W, H, bd)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 3, -1))
    try:
        dpb = [synth.noise_planes(rng, W, H, bd) for _ in range(4)] + [None, None]
        for s in range(4):
            vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(dpb[s])))
        dpb[4] = [p.copy() for p in dpb[0]]; dpb[5] = [p.copy() for p in dpb[0]]
        order = [4, 5, 0, 2, 1, 3]          # destination slots: later pictures overwrite the initial references
        for i, (db, sa, al) in enumerate(flagsets):
            dst = order[i % len(order)]
            pic = synth.gen_picture(rng, W, H, bd, dst_slot=dst, deblock=db, sao=sa, alf=al)
            want, dm_want = oracle_decompress(oracle, g, dpb[:4], pic)
            h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"]))
            assert h >= 0, b200.b200_last_error()
            dm = np.zeros((pic["ndmvr"] + 1, 2), np.int32)
            vvdec_b200.check(b200.b200_wait_picture(ctx, h, dm.ctypes.data, len(dm)))
            got = [np.zeros_like(p) for p in want]
            vvdec_b200.check(b200.b200_get_frame(ctx, dst, abi.plane_ptrs(got)))
            for c in range(3):
                assert np.array_equal(want[c], got[c]), f"picture {i} plane {c}: {len(np.argwhere(want[c] != got[c]))} diffs"
            assert np.array_equal(dm, dm_want)
            dpb[dst] = want
        assert b200.b200_ctx_kernel_launches(ctx) >= 5
    finally:
        b200.b200_ctx_destroy(ctx)


def test_ctx_errors(b200):
    ctx = C.c_void_p()
    for g, what in ((abi.make_geom(100, 64, 10), b"multiple of 8"), (abi.make_geom(64, 64, 7), b"bit depth"), (abi.make_geom(64, 64, 13), b"bit depth"),
                    (abi.make_geom(64, 64, 10, strides=(64, 32, 31)), b"stride")):
        assert b200.b200_ctx_create(C.byref(ctx), C.byref(g), 4, 2, -1) == -2, what
        assert what in b200.b200_last_error() and b"b200_ctx_create" in b200.b200_last_error()


def test_pic_upload_refuses_tables_and_boundaries(b200):
    """b200_pic_upload refuses the ALF table counts (a picture's tables may hold several slices' APS sets: up to 255 luma sets) and SAO virtual
    boundaries b200_alf_picture / b200_sao_picture refuse, before it copies anything; the same picture with the field restored decodes."""
    rng = np.random.default_rng(8)
    W, H, bd = 416, 240, 10
    g = abi.make_geom(W, H, bd)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        pic = synth.gen_picture(rng, W, H, bd, dst_slot=4)
        T, vb = pic["alfTabs"], abi.Vb()
        vb.numVer, vb.numHor, vb.posX[0], vb.posY[0] = 1, 1, 64, 120
        pic["struct"].vb = C.addressof(vb)
        def refused(what):
            return b200.b200_pic_upload(ctx, C.byref(pic["struct"])) == -2 and what in b200.b200_last_error() and b"b200_pic_upload" in b200.b200_last_error()
        n, cc = T.numLumaSets, T.numCc[0]
        for bad in (15, 256):
            T.numLumaSets = bad
            assert refused(b"numLumaSets"), bad
        T.numLumaSets = n
        T.numCc[0] = -1
        assert refused(b"numCc")
        T.numCc[0] = cc
        vb.posX[0] = 68
        assert refused(b"vertical virtual boundary")
        vb.posX[0], vb.posY[0] = 64, 244
        assert refused(b"horizontal virtual boundary")
        vb.posY[0] = 120
        h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"])); assert h >= 0, b200.b200_last_error()
        assert b200.b200_wait_picture(ctx, h, None, 0) == 0
    finally:
        b200.b200_ctx_destroy(ctx)


def test_invalid_records_are_reported(b200):
    """Records are validated on the device while they are bucketed: a PU pointing at a DPB slot the context does not have (or a TU with
    an impossible size) makes b200_pic_run / b200_decompress_picture refuse the picture with B200_ERR_PARAM."""
    rng = np.random.default_rng(5)
    W, H, bd = 416, 240, 10
    g = abi.make_geom(W, H, bd)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        ref = synth.noise_planes(rng, W, H, bd)
        for s in range(6): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(ref)))
        pic = synth.gen_picture(rng, W, H, bd, dst_slot=4, deblock=0, sao=0, alf=0)
        h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"])); assert h >= 0
        assert b200.b200_wait_picture(ctx, h, None, 0) == 0
        orig = pic["pus"]["refSlot"][3].copy()
        pic["pus"]["refSlot"][3] = (17, -1)
        assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and b"PU list" in b200.b200_last_error()
        pic["pus"]["refSlot"][3] = orig
        pic["tus"]["log2w"][0] = 7
        assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and b"TU list" in b200.b200_last_error()
        pic["tus"]["log2w"][0] = 2
        # records that would touch memory outside the picture or outside the uploaded arrays are refused too
        for arr, field, idx, bad, what in (("pus", "x", 5, W - 4 + 8, b"PU list"), ("pus", "y", 5, H, b"PU list"), ("pus", "x", 5, 2, b"PU list"),
                                           ("tus", "coefOff", 1, 1 << 30, b"TU list"), ("tus", "x", 1, W, b"TU list"), ("tus", "maxX", 1, 200, b"TU list")):
            keep = pic[arr][field][idx].copy()
            pic[arr][field][idx] = bad
            assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and what in b200.b200_last_error(), (arr, field)
            pic[arr][field][idx] = keep
        # fields the kernels index tables / working sets with (ADVICE r1): LFNST byte, joint-CbCr mode on a luma TU, transform-skip / BDPCM blocks wider than 32
        tus = pic["tus"]
        i_luma = int(np.flatnonzero((tus["comp"] == 0) & (tus["log2w"] >= 2) & (tus["log2h"] >= 2) & ((tus["flags"] & 7) == 0))[0])
        for field, bad in (("lfnst", 0x10), ("lfnst", 3), ("lfnst", 0x41), ("ict", 2)):
            keep = tus[field][i_luma].copy(); tus[field][i_luma] = bad
            assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and b"TU list" in b200.b200_last_error(), (field, bad)
            tus[field][i_luma] = keep
        keep = tus[i_luma].copy()
        tus["flags"][i_luma] |= 1; tus["log2w"][i_luma] = 6; tus["x"][i_luma] = 0                      # a 64-wide transform-skip block
        assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and b"TU list" in b200.b200_last_error()
        tus[i_luma] = keep
        tus["flags"][i_luma] |= 2                                                                      # BDPCM without transform skip / with a partial corner
        assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and b"TU list" in b200.b200_last_error()
        tus[i_luma] = keep
        fpic = synth.gen_picture(rng, W, H, bd, dst_slot=4)               # with filters: CTU records are range-checked too
        for arr, field, bad in (("alf", "lumaSet", 250), ("sao", "type", 7), ("alf", "ccIdx", 200)):
            recs = fpic["alf"]["ctus"] if arr == "alf" else fpic["sao"]
            keep = recs[0].copy()
            recs[field][0] = bad
            if arr == "alf": recs["enable"][0] = 1
            assert b200.b200_decompress_picture(ctx, C.byref(fpic["struct"])) == -2 and b"CTU record" in b200.b200_last_error(), (arr, field)
            recs[0] = keep
        h = b200.b200_decompress_picture(ctx, C.byref(fpic["struct"])); assert h >= 0
        assert b200.b200_wait_picture(ctx, h, None, 0) == 0
        dm = np.flatnonzero(pic["pus"]["flags"] & synth.PU_DMVR)
        if dm.size:
            keep = pic["pus"]["dmvrOff"][dm[0]].copy()
            pic["pus"]["dmvrOff"][dm[0]] = 1 << 30
            assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and b"PU list" in b200.b200_last_error()
            pic["pus"]["dmvrOff"][dm[0]] = keep
        h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"])); assert h >= 0      # the context is still usable
        assert b200.b200_wait_picture(ctx, h, None, 0) == 0
    finally:
        b200.b200_ctx_destroy(ctx)


@pytest.mark.parametrize("W,H,ctu,chroma_adj", [(416, 240, 128, True), (416, 240, 64, True), (832, 480, 128, False), (1920, 1080, 128, True)])
def test_lmcs_picture(b200, oracle, W, H, ctu, chroma_adj):
    """LMCS on (SURVEY 8 row a17): forward-mapped luma prediction fused into K2, luma TUs -> per-VPDU chroma scale -> scaled chroma
    TUs, inverse map before deblocking — against the oracle chain (which tests/test_lmcs_oracle_vs_ref.py pins to the real Reshape)."""
    _lmcs_pictures(b200, oracle, W, H, ctu, chroma_adj, 0.0, ["auto"])


@pytest.mark.parametrize("W,H,ctu,intra_frac", [(416, 240, 128, 0.15), (416, 240, 64, 1.0)])
def test_lmcs_picture_with_intra_cus(b200, oracle, W, H, ctu, intra_frac):
    """LMCS with intra and CIIP CUs: K6 runs twice on one list (luma blocks, then after the VPDU scales the chroma blocks, the luma blocks marked
    done), every picture under each kernel."""
    _lmcs_pictures(b200, oracle, W, H, ctu, True, intra_frac, ["v1", "v2"])


def _lmcs_pictures(b200, oracle, W, H, ctu, chroma_adj, intra_frac, kernels):
    rng = np.random.default_rng(W + ctu + int(100 * intra_frac))
    bd = 10
    g = abi.make_geom(W, H, bd, ctu=ctu)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        dpb = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
        for s in range(4): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(dpb[s])))
        for k in range(2):
            pic = synth.gen_picture(rng, W, H, bd, ctu=ctu, dst_slot=4 + k, lmcs=True, lmcs_chroma=chroma_adj, intra_frac=intra_frac)
            if intra_frac: assert len(pic["intraTus"]) and (pic["intraTus"]["comp"] > 0).any()
            want, dm_want = oracle_decompress(oracle, g, dpb, pic)
            for kernel in kernels:
                with intra_kernel(kernel): h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"]))
                assert h >= 0, b200.b200_last_error()
                dm = np.zeros((pic["ndmvr"] + 1, 2), np.int32)
                vvdec_b200.check(b200.b200_wait_picture(ctx, h, dm.ctypes.data, len(dm)))
                got = [np.zeros_like(p) for p in want]
                vvdec_b200.check(b200.b200_get_frame(ctx, 4 + k, abi.plane_ptrs(got)))
                for c in range(3):
                    assert np.array_equal(want[c], got[c]), f"{kernel}: picture {k} plane {c}: {len(np.argwhere(want[c] != got[c]))} diffs"
                assert np.array_equal(dm, dm_want)
    finally:
        b200.b200_ctx_destroy(ctx)


def test_weighted_prediction_picture(b200, oracle):
    """Explicit weighted prediction and GEO at picture level (together with LMCS: the combined luma is what gets forward-mapped)."""
    W, H, bd = 832, 480, 10
    rng = np.random.default_rng(31)
    g = abi.make_geom(W, H, bd)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        dpb = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
        for s in range(4): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(dpb[s])))
        for k, lm in enumerate((False, True)):
            pic = synth.gen_picture(rng, W, H, bd, dst_slot=4 + k, wp=True, lmcs=lm, pu_kw=dict(p_dmvr=0.0, p_bdof=0.0, p_bcw=0.3, p_geo=0.15))
            want, _ = oracle_decompress(oracle, g, dpb, pic)
            h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"])); assert h >= 0, b200.b200_last_error()
            vvdec_b200.check(b200.b200_wait_picture(ctx, h, None, 0))
            got = [np.zeros_like(p) for p in want]
            vvdec_b200.check(b200.b200_get_frame(ctx, 4 + k, abi.plane_ptrs(got)))
            for c in range(3):
                assert np.array_equal(want[c], got[c]), f"picture {k} plane {c}: {len(np.argwhere(want[c] != got[c]))} diffs"
    finally:
        b200.b200_ctx_destroy(ctx)


@pytest.mark.parametrize("W,H,ctu,intra_frac,seed", [(416, 240, 128, 0.25, 1), (416, 240, 64, 1.0, 2), (832, 480, 128, 0.15, 3), (1920, 1080, 128, 0.3, 4), (416, 240, 32, 1.0, 5)])
def test_picture_with_intra_cus(b200, oracle, W, H, ctu, intra_frac, seed):
    """Intra CUs reconstructed on the device inside the picture chain (SURVEY 8f-1, regular modes): K2 for the inter CUs, K1 (inter TUs reconstruct, TUs
    of intra CUs leave their residual in the residual planes), K6 over the intra blocks in decoding order — each reads the reconstruction of inter and
    earlier intra neighbours — then deblocking / SAO / ALF.  intra_frac 1.0 is an I picture.  Every picture is decoded under each K6 kernel in turn."""
    rng = np.random.default_rng(seed)
    bd = 10
    g = abi.make_geom(W, H, bd, ctu=ctu)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        dpb = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
        for s in range(4): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(dpb[s])))
        for i in range(2):
            pic = synth.gen_picture(rng, W, H, bd, ctu=ctu, dst_slot=4 + i, intra_frac=intra_frac)
            assert len(pic["intraTus"]) > 0 and (pic["tus"]["flags"] & abi.TU_RESI).any() and (pic["intraTus"]["flags"] & abi.INTRA_ADD_RESI).any()
            assert intra_frac == 1.0 or (pic["intraTus"]["ciip"] > 0).any()          # CIIP CUs among the inter CUs
            want, dm_want = oracle_decompress(oracle, g, dpb, pic)
            for kernel in ("v1", "v2"):
                with intra_kernel(kernel): h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"]))
                assert h >= 0, b200.b200_last_error()
                dm = np.zeros((pic["ndmvr"] + 1, 2), np.int32)
                vvdec_b200.check(b200.b200_wait_picture(ctx, h, dm.ctypes.data, len(dm)))
                got = [np.zeros_like(p) for p in want]
                vvdec_b200.check(b200.b200_get_frame(ctx, 4 + i, abi.plane_ptrs(got)))
                for c in range(3):
                    assert np.array_equal(want[c], got[c]), f"{kernel}: picture {i} plane {c}: {len(np.argwhere(want[c] != got[c]))} diffs"
                assert np.array_equal(dm, dm_want)
        # a record whose availability reaches outside the picture is refused
        bad = pic["intraTus"]; keep = bad[0].copy(); bad[0]["numAbove"] = 3; bad[0]["y"] = 0
        assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and b"intra block record" in b200.b200_last_error()
        bad[0] = keep
    finally:
        b200.b200_ctx_destroy(ctx)


def test_failed_host_register_does_not_resurface(b200, oracle):
    """b200_host_register on a range that is already registered fails, and the caller may go on with the memory unpinned (the glue's PinnedVec does).  That
    failure is reported once: the next picture on the same thread must not find it again in the CUDA runtime's per-thread last error."""
    rng = np.random.default_rng(9)
    W, H, bd = 416, 240, 10
    g = abi.make_geom(W, H, bd)
    refs = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
    pic = synth.gen_picture(rng, W, H, bd, dst_slot=4)
    want, _ = oracle_decompress(oracle, g, refs, pic)
    buf = np.zeros(1 << 16, np.uint8)
    assert b200.b200_host_register(buf.ctypes.data, buf.nbytes) == 0
    assert b200.b200_host_register(buf.ctypes.data, buf.nbytes) != 0         # already registered
    ctx = C.c_void_p()
    try:
        vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, 0))
        for s in range(4): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(refs[s])))
        h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"]))
        assert h >= 0, b200.b200_last_error()
        vvdec_b200.check(b200.b200_wait_picture(ctx, h, None, 0))
        got = [np.zeros_like(p) for p in want]
        vvdec_b200.check(b200.b200_get_frame(ctx, 4, abi.plane_ptrs(got)))
        for c in range(3): assert np.array_equal(want[c], got[c]), f"plane {c}"
    finally:
        b200.b200_ctx_destroy(ctx); b200.b200_host_unregister(buf.ctypes.data)


@pytest.mark.parametrize("kernel", ["auto", "v1", "v2"])
def test_intra_list_refusals(b200, oracle, kernel):
    """Intra lists the CTU-resident kernel cannot address are refused, and the context then decodes the next picture: a block that is not inside one
    CTU (b200_decompress_picture, before anything runs), and more than 3072 blocks in one CTU (overlapping records; only the CTU-resident kernel counts
    them, so b200_wait_picture reports it and the one-CTA-per-block kernel reconstructs the list)."""
    rng = np.random.default_rng(41)
    W, H, bd, ctu = 416, 240, 10, 64
    g = abi.make_geom(W, H, bd, ctu=ctu)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        dpb = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
        for s in range(4): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(dpb[s])))
        pic = synth.gen_picture(rng, W, H, bd, ctu=ctu, dst_slot=4, intra_frac=1.0)
        want, _ = oracle_decompress(oracle, g, dpb, pic)

        def decode_and_check():
            with intra_kernel(kernel): h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"]))
            assert h >= 0, b200.b200_last_error()
            vvdec_b200.check(b200.b200_wait_picture(ctx, h, None, 0))
            got = [np.zeros_like(p) for p in want]
            vvdec_b200.check(b200.b200_get_frame(ctx, 4, abi.plane_ptrs(got)))
            for c in range(3): assert np.array_equal(want[c], got[c]), f"plane {c}: {len(np.argwhere(want[c] != got[c]))} diffs"

        recs = pic["intraTus"]
        for comp, x, y, l2w, l2h in ((0, 56, 0, 4, 3), (0, 64, 60, 2, 3), (1, 24, 8, 4, 2), (2, 40, 28, 2, 3)):
            i = int(np.flatnonzero(recs["comp"] == comp)[0]); keep = recs[i].copy()
            recs[i]["x"], recs[i]["y"], recs[i]["log2w"], recs[i]["log2h"], recs[i]["numAbove"], recs[i]["numLeft"], recs[i]["flags"] = x, y, l2w, l2h, 0, 0, 0
            recs[i]["mode"], recs[i]["multiRefIdx"], recs[i]["mip"], recs[i]["ciip"] = 0, 0, 0, 0
            with intra_kernel(kernel):
                assert b200.b200_decompress_picture(ctx, C.byref(pic["struct"])) == -2 and b"intra block record" in b200.b200_last_error(), (comp, x, y)
            recs[i] = keep
        # the CCLM rows of tests.helpers.cclm_refusal_rows for this picture (CTU 64: no 64-wide chroma rows), each in place of a chroma record: the
        # device validator of the picture path refuses each
        i = int(np.flatnonzero(recs["comp"] == 1)[0]); keep = recs[i].copy()
        for name, bad, _ in cclm_refusal_rows(W, H, ctu)[2]:
            recs[i] = bad
            with intra_kernel(kernel):
                h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"]))
                rc = h if h < 0 else b200.b200_wait_picture(ctx, h, None, 0)
            assert rc == -2 and b"intra block record" in b200.b200_last_error(), (name, rc, b200.b200_last_error())
        recs[i] = keep
        decode_and_check()

        # one valid luma block repeated 3100 times, in the first CTU
        i = int(np.flatnonzero((recs["comp"] == 0) & (recs["x"] == 0) & (recs["y"] == 0))[0])
        many = np.ascontiguousarray(np.repeat(recs[i:i + 1], 3100))
        st = pic["struct"]; keep_ptr, keep_n = st.intraTus, st.numIntraTus
        st.intraTus, st.numIntraTus = many.ctypes.data, len(many)
        with intra_kernel(kernel): h = b200.b200_decompress_picture(ctx, C.byref(st))
        assert h >= 0, b200.b200_last_error()
        rc = b200.b200_wait_picture(ctx, h, None, 0)
        if kernel == "v1": assert rc == 0, b200.b200_last_error()
        else: assert rc == -2 and b"more than 3072" in b200.b200_last_error()
        st.intraTus, st.numIntraTus = keep_ptr, keep_n
        decode_and_check()
    finally:
        b200.b200_ctx_destroy(ctx)


def test_strided_copies_of_planes_that_start_in_a_registered_page(b200):
    """b200_ctx_load_slot_strided / b200_get_frame_strided with host planes whose first page the caller has registered for another array (cudaHostRegister
    pins whole pages; the glue pins its work-list vectors, which share the heap with the picture buffers): the planes run past that registration, and the
    copies still move every sample."""
    rng = np.random.default_rng(12)
    W, H, bd, margin = 416, 240, 10, 16
    g = abi.make_geom(W, H, bd)
    page = 4096
    want = synth.noise_planes(rng, W, H, bd)
    bufs, planes, outs = [], [], []
    for c, p in enumerate(want):
        h, w = p.shape
        raw = np.zeros(2 * page + (h * (w + margin) + page) * 2, np.uint8)
        base = (-raw.ctypes.data) % page                          # a page-aligned page, then the plane starting inside the next one
        assert b200.b200_host_register(raw.ctypes.data + base, page) == 0
        bufs.append((raw, raw.ctypes.data + base))
        off = base + page - 64 if c == 0 else base + 256                  # luma: the registered page's last 64 bytes; chroma: near its start
        view = raw[off:off + h * (w + margin) * 2].view(np.int16).reshape(h, w + margin)
        view[:, :w] = p; planes.append(view)
    ctx = C.c_void_p()
    try:
        vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 2, 2, -1))
        strides = (C.c_ssize_t * 3)(*(v.shape[1] for v in planes))
        vvdec_b200.check(b200.b200_ctx_load_slot_strided(ctx, 0, abi.plane_ptrs(planes), strides))
        got = [np.zeros_like(p) for p in want]
        vvdec_b200.check(b200.b200_get_frame(ctx, 0, abi.plane_ptrs(got)))
        for c in range(3): assert np.array_equal(got[c], want[c]), f"load plane {c}"
        for v in planes: v[...] = 0
        vvdec_b200.check(b200.b200_get_frame_strided(ctx, 0, abi.plane_ptrs(planes), strides))
        for c in range(3): assert np.array_equal(planes[c][:, :want[c].shape[1]], want[c]), f"get plane {c}"
    finally:
        if ctx: b200.b200_ctx_destroy(ctx)
        for raw, ptr in bufs: b200.b200_host_unregister(ptr)


@pytest.mark.parametrize("name,lmcs", [("shapes_10bit", True), ("wp_10bit", True), ("edges_ctu32_stride_odd", False)])
def test_designed_mc_lists_in_a_picture(b200, oracle, name, lmcs):
    """Lists of the designed K2 sweep (synth.mc_sweep) through b200_decompress_picture, K2 reading the device DPB slots: with LMCS every luma store site
    (uni, bi, BDOF, DMVR, affine uni / bi, GEO; weighted uni / bi / affine in the wp list) forward-maps; the edges list runs in a context with CTU 32 and
    an odd luma stride.  Samples and the DMVR deltas b200_wait_picture returns match the oracle chain; the samples no PU covers come from `given`."""
    from tests.helpers import mc_dst
    case = synth.mc_sweep(name)
    g, W, H, bd = case["g"], case["W"], case["H"], case["bd"]
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        for s in range(4): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(case["refs"][s])))
        pic = synth.gen_picture(np.random.default_rng(9), W, H, bd, ctu=case["ctu"], dst_slot=4, inter=False, tu_kw=dict(p_cbf=0.0), deblock=False, sao=False,
                                alf=False, lmcs=lmcs)
        st = pic["struct"]
        pic["pus"], pic["ndmvr"] = case["pus"], case["ndmvr"]
        st.pus = case["pus"].ctypes.data; st.numPus = len(case["pus"]); st.numDmvr = case["ndmvr"] + 1
        pic["given"] = mc_dst(g, 0)
        for c in range(3): st.given[c] = pic["given"][c].ctypes.data
        if case["wp"]:
            pic["wp"] = case["wp"][1]; st.wp = pic["wp"].ctypes.data; st.numWp = len(pic["wp"])
        want, dm_want = oracle_decompress(oracle, g, case["refs"], pic)
        h = b200.b200_decompress_picture(ctx, C.byref(st))
        assert h >= 0, b200.b200_last_error()
        dm = np.zeros_like(dm_want)
        vvdec_b200.check(b200.b200_wait_picture(ctx, h, dm.ctypes.data, len(dm)))
        got = mc_dst(g, 0)
        vvdec_b200.check(b200.b200_get_frame(ctx, 4, abi.plane_ptrs(got)))
        for c in range(3):
            w, hh = (W, H) if c == 0 else (W // 2, H // 2)
            bad = np.argwhere(want[c][:hh, :w] != got[c][:hh, :w])
            assert len(bad) == 0, f"{name}: plane {c}: {len(bad)} diffs, first at {bad[:1].tolist()}"
        assert np.array_equal(dm, dm_want), f"{name}: DMVR deltas differ"
        if lmcs and name == "shapes_10bit": assert {t for t in case["tags"]} >= {"uni0", "bi", "bdof", "dmvr", "aff4_uni", "aff4_bi", "geo"}
    finally:
        b200.b200_ctx_destroy(ctx)


def test_work_lists_and_dmvr_deltas_in_arrays_that_start_in_a_registered_page(b200, oracle):
    """b200_decompress_picture reads the PU list from, and b200_wait_picture writes the DMVR deltas into, host arrays that start in the last bytes of a page
    the caller registered for another array and run past it (the layout the glue's pinned work-list vectors can give the decoder's own arrays): both
    copies still move every byte."""
    rng = np.random.default_rng(13)
    W, H, bd = 416, 240, 10
    g = abi.make_geom(W, H, bd)
    dpb = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
    pic = synth.gen_picture(rng, W, H, bd, dst_slot=4, deblock=False, sao=False, alf=False, pu_kw=dict(p_dmvr=0.9, p_bi=0.9, mv_sigma=2.0))
    want, dm_want = oracle_decompress(oracle, g, dpb, pic)
    assert (dm_want != 0).any() and len(dm_want) * 8 > 64
    page = 4096
    raw = np.zeros(2 * page + len(dm_want) * 8 + page, np.uint8)
    base = (-raw.ctypes.data) % page
    rawp = np.zeros(2 * page + pic["pus"].nbytes + page, np.uint8)
    basep = (-rawp.ctypes.data) % page
    assert b200.b200_host_register(raw.ctypes.data + base, page) == 0
    assert b200.b200_host_register(rawp.ctypes.data + basep, page) == 0
    pus = rawp[basep + page - 64:basep + page - 64 + pic["pus"].nbytes].view(synth.PU_DTYPE)
    pus[:] = pic["pus"]; pic["struct"].pus = pus.ctypes.data
    ctx = C.c_void_p()
    try:
        vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
        for s in range(4): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(dpb[s])))
        dm = raw[base + page - 64:base + page - 64 + dm_want.size * 4].view(np.int32).reshape(dm_want.shape)
        h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"])); assert h >= 0, b200.b200_last_error()
        vvdec_b200.check(b200.b200_wait_picture(ctx, h, dm.ctypes.data, len(dm)))
        assert np.array_equal(dm, dm_want)
        got = [np.zeros_like(p) for p in want]
        vvdec_b200.check(b200.b200_get_frame(ctx, 4, abi.plane_ptrs(got)))
        for c in range(3): assert np.array_equal(got[c], want[c]), f"plane {c}"
    finally:
        if ctx: b200.b200_ctx_destroy(ctx)
        b200.b200_host_unregister(raw.ctypes.data + base); b200.b200_host_unregister(rawp.ctypes.data + basep)


@pytest.mark.parametrize("name,strides", [("tight_spacing", None), ("ctu_edges_ctu32_200x136", (201, 103, 100)), ("qp_ladf_10bit", None)])
def test_designed_deblocking_in_a_picture(b200, oracle, name, strides):
    """Cases of the designed K3 sweep (synth.lf_sweep) through b200_decompress_picture: the designed planes as `given`, no PUs or TUs, deblocking on with
    the case's grids, slices and LADF; the CTU-32 case with an odd luma stride.  The frame equals the oracle chain's."""
    case = synth.lf_sweep(name)
    W, H, bd, ctu = case["W"], case["H"], case["bd"], case["ctu"]
    g = abi.make_geom(W, H, bd, ctu=ctu, strides=strides)
    given = []
    for c in range(3):
        w, h = (W, H) if c == 0 else (W // 2, H // 2)
        p = np.zeros((h, g.stride[c]), np.int16); p[:, :w] = case["planes"][c][:, :w]; given.append(p)
    pic = synth.gen_picture(np.random.default_rng(3), W, H, bd, ctu=ctu, dst_slot=4, inter=False, tu_kw=dict(p_cbf=0.0), deblock=False, sao=False, alf=False)
    st = pic["struct"]
    assert len(pic["pus"]) == 0 and len(pic["tus"]) == 0
    pic["given"] = given
    for c in range(3): st.given[c] = given[c].ctypes.data
    pic["lfV"], pic["lfH"], pic["lfSlices"], pic["lfSeq"] = case["lfV"], case["lfH"], case["slices"], case["seq"]
    st.flags |= abi.PIC_DEBLOCK; st.lfV = case["lfV"].ctypes.data; st.lfH = case["lfH"].ctypes.data
    st.lfSlices = case["slices"].ctypes.data; st.numLfSlices = len(case["slices"]); st.lfSeq = C.addressof(case["seq"])
    if case["ctuSlice"] is not None: pic["ctuSlice"] = case["ctuSlice"]; st.ctuSlice = case["ctuSlice"].ctypes.data
    refs = [[np.zeros_like(p) for p in given] for _ in range(4)]
    want, _ = oracle_decompress(oracle, g, refs, pic)
    assert not np.array_equal(want[0], given[0])
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        h = b200.b200_decompress_picture(ctx, C.byref(st))
        assert h >= 0, b200.b200_last_error()
        vvdec_b200.check(b200.b200_wait_picture(ctx, h, None, 0))
        got = [np.zeros_like(p) for p in given]
        vvdec_b200.check(b200.b200_get_frame(ctx, 4, abi.plane_ptrs(got)))
        for c in range(3):
            w, hh = (W, H) if c == 0 else (W // 2, H // 2)
            bad = np.argwhere(want[c][:hh, :w] != got[c][:hh, :w])
            assert len(bad) == 0, f"{name}: plane {c}: {len(bad)} diffs, first at {bad[:1].tolist()}"
    finally:
        b200.b200_ctx_destroy(ctx)


def _filter_picture(b200, oracle, case, strides, sao, alf, flags=abi.PIC_SAO | abi.PIC_ALF, bd=None):
    """A designed K4 / K5 sweep picture through b200_decompress_picture: its planes as `given`, no PUs or TUs, SAO and / or ALF on with the given
    records.  Returns the handle's error (or None) and, when it decoded, whether the frame equals the oracle chain's on the plane width."""
    W, H, ctu = case["W"], case["H"], case["ctu"]
    bd = bd or case["bd"]
    g = abi.make_geom(W, H, bd, ctu=ctu, strides=strides)
    given = []
    for c in range(3):
        w, h = (W, H) if c == 0 else (W // 2, H // 2)
        p = np.zeros((h, g.stride[c]), np.int16); p[:, :w] = case["planes"][c][:, :w]; given.append(p)
    pic = synth.gen_picture(np.random.default_rng(3), W, H, bd, ctu=ctu, dst_slot=4, inter=False, tu_kw=dict(p_cbf=0.0), deblock=False, sao=False, alf=False)
    st = pic["struct"]
    pic["given"] = given
    for c in range(3): st.given[c] = given[c].ctypes.data
    T = abi.make_alf_tables(alf)
    pic["sao"], pic["alf"], pic["alfTabs"] = sao, dict(ctus=alf["ctus"]), T
    st.flags |= flags; st.sao = sao.ctypes.data; st.alf = alf["ctus"].ctypes.data; st.alfTabs = C.addressof(T)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        h = b200.b200_decompress_picture(ctx, C.byref(st))
        if h < 0: return b200.b200_last_error(), None
        vvdec_b200.check(b200.b200_wait_picture(ctx, h, None, 0))
        got = [np.zeros_like(p) for p in given]
        vvdec_b200.check(b200.b200_get_frame(ctx, 4, abi.plane_ptrs(got)))
    finally:
        b200.b200_ctx_destroy(ctx)
    want, _ = oracle_decompress(oracle, g, [[np.zeros_like(p) for p in given] for _ in range(4)], pic)
    for c in range(3):
        w, hh = (W, H) if c == 0 else (W // 2, H // 2)
        bad = np.argwhere(want[c][:hh, :w] != got[c][:hh, :w])
        if len(bad): return None, f"{case['name']}: plane {c}: {len(bad)} diffs, first at {bad[:1].tolist()}"
    return None, True


@pytest.mark.parametrize("kind,name,strides", [("alf", "ccalf_10bit_ctu32", None), ("alf", "coeffs_10bit_ctu32_last24", (280, 136, 140)),
                                               ("sao", "avail_masks_ctu32", None)])
def test_designed_sao_alf_in_a_picture(b200, oracle, kind, name, strides):
    """Cases of the designed K4 / K5 sweeps through b200_decompress_picture with SAO and ALF on: CC-ALF clipping both ways; CTU 32 with the ALF virtual
    boundary rows at the picture bottom and padded strides; every SAO avail mask.  The other filter's records come from gen_sao / gen_alf.  The frame
    equals the oracle chain's."""
    rng = np.random.default_rng(11)
    case = synth.alf_sweep(name) if kind == "alf" else synth.sao_sweep(name)
    W, H, ctu = case["W"], case["H"], case["ctu"]
    sao = case["ctus"] if kind == "sao" else synth.gen_sao(rng, W, H, ctu, case["bd"], p_on=0.5)
    alf = case["tables"] if kind == "alf" else synth.gen_alf(rng, W, H, ctu, case["bd"], n_aps=2)
    err, ok = _filter_picture(b200, oracle, case, strides, sao, alf)
    assert err is None and ok is True, (err, ok)


@pytest.mark.parametrize("what,bad,fixed", [("ALF at 12 bit", dict(bd=12), dict(bd=10)), ("SAO with a Cb stride of 4k + 2", dict(strides=(264, 134, 132)), dict(strides=(264, 136, 132)))])
def test_sao_alf_picture_refusals(b200, oracle, what, bad, fixed):
    """b200_decompress_picture refuses ALF above 10 bit and SAO / ALF with a plane stride that is not a multiple of 4 before any device work; the same
    picture with the field fixed decodes and equals the oracle chain's."""
    case = synth.sao_sweep("eo_8bit_ctu32_partial")
    rng = np.random.default_rng(12)
    alf = synth.gen_alf(rng, case["W"], case["H"], case["ctu"], 10, n_aps=2)
    flags = abi.PIC_ALF if "bd" in bad else abi.PIC_SAO
    err, ok = _filter_picture(b200, oracle, case, bad.get("strides"), case["ctus"], alf, flags=flags, bd=bad.get("bd", 10))
    assert err is not None and b"b200_pic_upload" in err, (what, err, ok)
    err, ok = _filter_picture(b200, oracle, case, fixed.get("strides"), case["ctus"], alf, flags=flags, bd=fixed.get("bd", 10))
    assert err is None and ok is True, (what, err, ok)


@pytest.mark.parametrize("ctu", [32, 64, 128])
def test_k1_lmcs_chroma_scaling_in_a_picture(b200, oracle, ctu):
    """K1's LMCS passes on the picture path (luma TUs, then the per-VPDU chroma scale, then chroma TUs scaled by their VPDU's entry; blocks of 4 samples
    unscaled, joint-CbCr partners scaled): synth.k1_lmcs_picture's TUs over a `given` prediction, no PUs, deblocking / SAO / ALF off.  The VPDUs use at
    least three different scales besides the neutral one, and the picture matches the oracle chain."""
    W, H, bd = 256, 128, 10
    g = abi.make_geom(W, H, bd, ctu=ctu)
    tus, coefs, given, tags = synth.k1_lmcs_picture(ctu, W, H, bd)
    pic = synth.gen_picture(np.random.default_rng(ctu), W, H, bd, ctu=ctu, dst_slot=4, inter=False, tu_kw=dict(p_cbf=0.0), deblock=False, sao=False,
                            alf=False, lmcs=True)
    st = pic["struct"]
    assert st.flags == abi.PIC_LMCS and pic["lmcs"]["struct"].chromaAdj
    pic["tus"], pic["coefs"], pic["given"] = tus, coefs, given
    st.tus, st.numTus, st.coefs, st.numCoefs = tus.ctypes.data, len(tus), coefs.ctypes.data, len(coefs)
    for c in range(3): st.given[c] = given[c].ctypes.data
    # the VPDU scales the chroma TUs see: the luma plane after the luma TUs
    luma = [given[0].copy(), None, None]
    ly = np.ascontiguousarray(tus[tus["comp"] == 0])
    oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(luma), ly.ctypes.data, len(ly), coefs, None, 0)
    vs = 64 if ctu == 128 else ctu
    scale = np.zeros((W // vs) * (H // vs), np.int32)
    oracle.orc_lmcs_vpdu_scales(C.byref(g), luma[0], C.byref(pic["lmcs"]["struct"]), scale.ctypes.data)
    assert len(set(scale.tolist()) - {2048}) >= 3, scale
    dpb = [[np.zeros_like(p) for p in given] for _ in range(4)]
    want, _ = oracle_decompress(oracle, g, dpb, pic)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        h = b200.b200_decompress_picture(ctx, C.byref(st))
        assert h >= 0, b200.b200_last_error()
        vvdec_b200.check(b200.b200_wait_picture(ctx, h, None, 0))
        got = [np.zeros_like(p) for p in want]
        vvdec_b200.check(b200.b200_get_frame(ctx, 4, abi.plane_ptrs(got)))
        for c in range(3):
            bad = np.argwhere(want[c] != got[c])
            assert len(bad) == 0, f"CTU {ctu}: plane {c}: {len(bad)} diffs, first at {bad[:1].tolist()}"
    finally:
        b200.b200_ctx_destroy(ctx)


def test_slice_map_without_deblocking_in_a_reused_arena(b200, oracle):
    """A picture of several slices with deblocking off still carries its CTU slice map (the glue passes one whenever there is more than one slice); the
    map is only read by deblocking, so it is neither uploaded nor checked.  The picture runs in the one arena right after a picture with the same work
    lists and deblocking on: where its map entry lies, the arena still holds that picture's vertical edge grid, bytes far past the slice count.  It
    decodes and equals the oracle chain's frame."""
    W, H, bd = 416, 240, 10
    g = abi.make_geom(W, H, bd)
    rng = np.random.default_rng(12)
    refs = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
    nctu = ((W + 127) // 128) * ((H + 127) // 128)
    first = synth.gen_picture(rng, W, H, bd, dst_slot=4, sao=False, alf=False)
    first["lfSlices"] = np.zeros(4, synth.LFSLICE_DTYPE); first["ctuSlice"] = (np.arange(nctu) % 4).astype(np.uint8)
    st = first["struct"]; st.lfSlices = first["lfSlices"].ctypes.data; st.numLfSlices = 4; st.ctuSlice = first["ctuSlice"].ctypes.data
    # the same lists without deblocking: the two grid entries shrink to 256 bytes each, so the map entry starts 512 bytes into the first picture's lfV
    assert first["lfV"].reshape(-1).view(np.uint8)[512:512 + nctu].max() >= 2
    second = {k: first[k] for k in ("pus", "ndmvr", "tus", "coefs")}
    second["sao"] = synth.gen_sao(rng, W, H, 128, bd, p_on=0.5)
    second["ctuSlice"] = (np.arange(nctu) % 2).astype(np.uint8); second["lfSlices"] = np.zeros(2, synth.LFSLICE_DTYPE)
    st = abi.Picture.from_buffer_copy(st); second["struct"] = st
    st.dstSlot = 5; st.flags = abi.PIC_SAO; st.sao = second["sao"].ctypes.data
    st.ctuSlice = second["ctuSlice"].ctypes.data; st.lfSlices = second["lfSlices"].ctypes.data; st.numLfSlices = 2
    want, _ = oracle_decompress(oracle, g, refs, second)
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 1, -1))
    try:
        for s in range(4): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(refs[s])))
        for pic in (first, second):
            h = b200.b200_decompress_picture(ctx, C.byref(pic["struct"]))
            assert h == 0, b200.b200_last_error()
            vvdec_b200.check(b200.b200_wait_picture(ctx, h, None, 0))
        got = [np.zeros_like(p) for p in want]
        vvdec_b200.check(b200.b200_get_frame(ctx, 5, abi.plane_ptrs(got)))
        for c in range(3): assert np.array_equal(got[c], want[c]), f"plane {c}"
    finally:
        b200.b200_ctx_destroy(ctx)
