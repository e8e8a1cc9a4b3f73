"""The DecLibRecon seam from a real BITSTREAM, on the GPU (SURVEY 8c level L2, row f-4; VERDICT r1 item 1 "execute the seam").

A VVC stream written by oracle/vvc_stream.py (see tests/test_stream_cpu.py) is decoded twice through the reference's public API (vvdec_decode / vvdec_flush):
by the stock library, and by the same library with b200glue::DecLibReconB200 compiled in behind the DecLibRecon seam (oracle/_ref/libvvdec_swapped.so,
swap_recon.h) — parser, DecLib scheduling, picture list and output of the reference; reconstruction on the device through the C ABI.  All output frames must
be bit-exact.  (Runs last among the GPU tests: the file name sorts behind test_seam_gpu.py.  The device decode of every case runs in a child process with a time limit,
so a crash or a hang fails one case.)"""
import os, numpy as np, pytest
from oracle import vvc_stream as vs
from tests import test_stream_cpu
from tests.test_stream_cpu import ALL, INTRA, SL3, gop4, gop8, low_delay, _diff, _mixed_slice_types, _weighted

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (vs.available() and os.path.exists(vs.SWAP_SO)), reason="oracle/_ref not built")]

CASES = {
    "I_all_intra_tools": (dict(INTRA, width=416, height=240), lambda: [vs.Pic(0), vs.Pic(1, idr=True)]),
    "I_dual_tree_ctu128": (dict(INTRA, width=416, height=240, ctu=128, dual_tree=True), lambda: [vs.Pic(0)]),
    "gop_all_tools": (dict(ALL, width=416, height=240), gop4),
    "gop_all_tools_ctu128": (dict(ALL, width=416, height=240, ctu=128), gop4),
    "gop_ctu32": (dict(ALL, width=256, height=128, ctu=32, max_bt_inter=32, max_tt_inter=32), gop4),
    "gop_cu_qp_delta": (dict(ALL, width=256, height=128, cu_qp_delta=True), gop4),
    "low_delay_8": (dict(ALL, width=416, height=240), lambda: low_delay(8)),
    "gop8_x2": (dict(ALL, width=416, height=240, dpb_size=8), lambda: gop8(n_gops=2)),
    "gop_alf_ccalf_lmcs": (dict(ALL, width=416, height=240, alf=True, ccalf=True, lmcs=True), lambda: vs.with_lmcs(vs.with_alf(gop4(), np.random.default_rng(4)), np.random.default_rng(5))),
    "gop_max_transform_32": (dict(ALL, width=416, height=240, max_tb64=False), gop4),
    "gop_intra_slice_in_inter_pictures": (dict(ALL, **SL3), _mixed_slice_types),
    "gop_3slices_alf_lmcs_no_lf_across": (dict(ALL, **SL3, alf=True, ccalf=True, lmcs=True, lf_across_slices=False),
                                          lambda: vs.with_lmcs(vs.with_alf(gop4(), np.random.default_rng(11)), np.random.default_rng(12))),
    "gop_weighted_prediction": (dict(ALL, width=416, height=240, weighted_pred=True, weighted_bipred=True), lambda: _weighted(gop4())),
    "low_delay_alf_lmcs": (dict(ALL, width=416, height=240, alf=True, ccalf=True, lmcs=True), lambda: vs.with_lmcs(vs.with_alf(low_delay(6), np.random.default_rng(7)), np.random.default_rng(8), every=2)),
    # the glue's device mode on 4:0:0, 8 bit, CTU 32, a picture size that is not a multiple of the CTU, tiles, scaling lists with three slices, intra pictures
    # inside a low-delay stream (the CPU cases as they are)
    **{n: test_stream_cpu.CASES[n] for n in ("gop_monochrome_lmcs_alf", "gop_ctu32_8bit", "gop_picture_not_ctu_aligned", "gop_4tiles_no_lf_across_alf",
                                             "gop_alf_lmcs_8bit", "gop_scaling_lists_3slices_lmcs", "low_delay_with_intra_pictures")},
}


@pytest.mark.parametrize("name", list(CASES))
def test_stream_stock_vs_device_decoder(name):
    from tests import stream_util as su
    kw, pics = CASES[name]
    aus, drawn, _ = vs.build_stream(vs.Config(**kw), pics(), seed=3 + len(name))
    stock = vs.decode(vs.REF_SO, aus, threads=4)
    assert _diff(drawn, stock) == [0] * len(aus)
    got, _ = su.decode_swapped_device_guarded(aus, threads=4)
    assert _diff(got, stock) == [0] * len(aus)


def test_long_stream_on_the_device():
    """five GOPs: picture recycling in the reference's PicListManager, slot turnover in the device DPB, two recon instances alternating"""
    from tests import stream_util as su
    pics = []
    for k in range(5): pics += gop4(4 * k, idr=(k == 0))[(0 if k == 0 else 1):]
    aus, drawn, _ = vs.build_stream(vs.Config(**dict(ALL, width=256, height=128)), pics, seed=9)
    stock = vs.decode(vs.REF_SO, aus, threads=4)
    got, _ = su.decode_swapped_device_guarded(aus, threads=4)
    assert _diff(got, stock) == [0] * len(aus)


def test_new_sequence_with_another_geometry_on_the_device():
    """an IDR with new parameter sets (picture size, CTU size, bit depth): the class rebuilds its device context (DecLibReconB200::preparePicture)"""
    from tests import stream_util as su
    from tests.test_stream_cpu import sequence_change_stream
    aus, drawn = sequence_change_stream()
    stock = vs.decode(vs.REF_SO, aus, threads=4, frame_samples=256 * 192 * 2)
    got, _ = su.decode_swapped_device_guarded(aus, threads=4, frame_samples=256 * 192 * 2)
    assert _diff(got, stock) == [0] * len(aus)


def test_hash_sei_with_parse_delay_0_on_the_device():
    """decoded-picture-hash SEIs with one thread (parseFrameDelay 0): the parser waits for pic->reconDone on the API thread, the class completes the picture from a pool
    task (setAsyncFinish); the decoder verifies the hashes of what came back from the device itself"""
    from tests import stream_util as su
    aus, drawn, _ = vs.build_stream(vs.Config(**dict(ALL, width=416, height=240)), gop4(), seed=4, hash_sei="md5")
    stock = vs.decode(vs.REF_SO, aus, threads=1)
    assert vs.decode.hash_errors == 0
    got, hash_errors = su.decode_swapped_device_guarded(aus, threads=1, async_finish=True, timeout=180)
    assert hash_errors == 0 and _diff(got, stock) == [0] * len(aus)


@pytest.mark.parametrize("seed", [2003, 2017, 2130, 3179, 5001, 5014])
def test_random_streams_on_the_device(seed):
    """the fuzz draws of test_stream_cpu.test_random_streams on the device: the same thread count, hash SEIs and completion by a pool task on odd seeds"""
    from tests import stream_util as su
    kw, pics, _ = su._stream_fuzz().random_case(seed)
    aus, drawn, _ = vs.build_stream(vs.Config(**kw), pics, seed=seed, hash_sei="md5" if seed & 1 else None)
    stock = vs.decode(vs.REF_SO, aus)
    assert _diff(drawn, stock) == [0] * len(aus)
    got, hash_errors = su.decode_swapped_device_guarded(aus, threads=1 + 3 * (seed % 3 == 0), async_finish=bool(seed & 1))
    assert hash_errors == 0 and _diff(got, stock) == [0] * len(aus)
