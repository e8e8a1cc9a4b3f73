"""Edge grids derived on the H100 from CU / TU records (B200_PIC_DERIVE_LF, csrc/lf_derive.cu) against the reference's own derivation.

  * b200_lf_derive (the kernel-level entry point, same launches as the picture path) on the records of tests/golden/lf_derive_pictures.npz and — where
    oracle/_ref holds a build of the current glue — on the records the drop-in class emits for seam pictures: the grids read back equal what
    calcFilterStrengthsCTU + flattenLfCtu give for the same pictures, byte for byte; a slice with deblocking disabled ends its CTUs.
  * The drop-in class with the derivation switched on (B200_LF_DERIVE=1) on the device: seam pictures and bitstreams decode to the stock decoder's frames,
    with the streams' decoded-picture hash SEIs verified.
  * A bad record makes b200_pic_run return B200_ERR_PARAM before anything runs."""
import ctypes as C
import os
import numpy as np
import pytest
from tests import helpers
from tests.test_lf_derive_cpu import (CASES, SIZES, GOLDEN_NAMES, built_with_derivation, check_grids, flatten_grids, first_difference, golden, lf_derive,
                                      needs_glue, records_of, with_disabled_slice)
from vvdec_b200 import abi

ref = helpers.load_ref()
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_device_grids_of_the_golden_pictures(name):
    import vvdec_b200
    lib = vvdec_b200.lib()
    g, r, wantV, wantH = next((c[1], c[2], c[3], c[4]) for c in golden() if c[0] == name)
    rc, V, H = lf_derive(lib.b200_lf_derive, g, r)
    assert rc == 0, lib.b200_last_error()
    check_grids(g, (wantV, wantH), (V, H))


@needs_glue
@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_grids_equal_calc_filter_strengths(name, size):
    import vvdec_b200
    lib = vvdec_b200.lib()
    case = helpers.SeamCase(ref, np.random.default_rng(3), *SIZES[size], **CASES[name])
    wantV, wantH, _ = flatten_grids(case, False)
    _, _, flat = flatten_grids(case, True)
    rc, V, H = lf_derive(lib.b200_lf_derive, case.g, records_of(flat, case.g))
    assert rc == 0, lib.b200_last_error()
    W4 = case.g.width >> 2
    for k, want, got in (("lfV", wantV, V), ("lfH", wantH, H)):
        assert want.tobytes() == got.tobytes(), f"{k}: {first_difference(want, got, W4)}"


def run_device(case, derive):
    old = os.environ.get("B200_LF_DERIVE")
    os.environ["B200_LF_DERIVE"] = "1" if derive else "0"
    try: return case.run_b200()
    finally:
        if old is None: del os.environ["B200_LF_DERIVE"]
        else: os.environ["B200_LF_DERIVE"] = old


@needs_glue
@pytest.mark.parametrize("name", sorted(CASES))
def test_seam_pictures_on_the_device_equal_the_stock_decoder(name):
    case = helpers.SeamCase(ref, np.random.default_rng(7), 416, 240, **CASES[name])
    want, _, _ = case.run_stock()
    got, _, secs = run_device(case, True)
    assert secs >= 0, f"the device path failed ({secs})"
    for c in range(3):
        assert np.array_equal(want[c], got[c]), f"plane {c}: {np.count_nonzero(want[c] != got[c])} samples differ from the stock DecLibRecon"


STREAMS = ["gop_all_tools", "gop_ctu32_8bit", "I_dual_tree_ctu128", "gop_4slices_no_lf_across_deblock_override", "gop_ladf_chroma_deblock_offsets", "gop_monochrome_lmcs_alf", "gop_picture_not_ctu_aligned",
           "gop_4tiles_no_lf_across_alf", "low_delay_8", "gop_no_deblocking"]


@pytest.mark.parametrize("name", STREAMS)
def test_streams_on_the_device_with_derivation(name):
    from oracle import vvc_stream as vs
    from tests import stream_util as su
    from tests.test_stream_cpu import _diff
    if not (vs.available() and built_with_derivation(vs.SWAP_SO)): pytest.skip("oracle/_ref/libvvdec_swapped.so is not built from the current glue")
    aus, pics, samples, _ = su.corpus_stream(f"{name}-s1")
    stock = vs.decode(vs.REF_SO, aus, frame_samples=samples)
    os.environ["B200_LF_DERIVE"] = "1"                                      # inherited by the decoding child process
    try: got, hash_errors = su.decode_swapped_device_guarded(aus, threads=4, frame_samples=samples)
    finally: del os.environ["B200_LF_DERIVE"]
    assert hash_errors == 0
    assert _diff(got, stock) == [0] * len(stock)


def test_bad_record_is_refused_before_anything_runs():
    import vvdec_b200
    lib = vvdec_b200.lib()
    g, r = next((c[1], c[2]) for c in golden() if c[0].startswith("B_5slices"))
    r = {k: v.copy() for k, v in r.items()}
    r["cus"][int(r["ctuCus"][1])]["x"] = 0                                  # a CU listed under the second CTU that lies in the first
    p = abi.Picture()
    p.dstSlot = 4; p.flags = abi.PIC_DEBLOCK | abi.PIC_DERIVE_LF                 # (no PUs: only the edge derivation's records are under test)
    p.lfSlices, p.numLfSlices = r["slices"].ctypes.data, len(r["slices"])
    p.lfCus, p.numLfCus, p.lfTus, p.numLfTus = r["cus"].ctypes.data, len(r["cus"]), r["tus"].ctypes.data, len(r["tus"])
    p.lfCtuCus, p.lfSliceB = r["ctuCus"].ctypes.data, r["sliceB"].ctypes.data
    ctx = C.c_void_p()
    vvdec_b200.check(lib.b200_ctx_create(C.byref(ctx), C.byref(g), 17, 2, 0))
    try:
        n0 = lib.b200_ctx_kernel_launches(ctx)
        h = lib.b200_pic_upload(ctx, C.byref(p))
        assert h >= 0, lib.b200_last_error()
        n1 = lib.b200_ctx_kernel_launches(ctx)
        assert lib.b200_pic_run(ctx, h) == -2
        assert b"edge derivation" in lib.b200_last_error()
        assert lib.b200_ctx_kernel_launches(ctx) == n1 > n0                 # the upload's checks ran, the picture's kernels did not
    finally:
        lib.b200_ctx_destroy(ctx)


@pytest.mark.parametrize("disabled", [1, 2])
def test_slice_with_deblocking_disabled_ends_its_ctus(disabled):
    """Raster slices that start inside CTU rows (the golden three-slice picture): see test_lf_derive_cpu.with_disabled_slice."""
    import vvdec_b200
    lib = vvdec_b200.lib()
    g, r, wantV, wantH = next((c[1], c[2], c[3], c[4]) for c in golden() if c[0].startswith("B_3slices"))
    r, wantV, wantH, cut = with_disabled_slice(g, r, wantV, wantH, disabled)
    assert cut > 0
    rc, V, H = lf_derive(lib.b200_lf_derive, g, r)
    assert rc == 0, lib.b200_last_error()
    check_grids(g, (wantV, wantH), (V, H))
