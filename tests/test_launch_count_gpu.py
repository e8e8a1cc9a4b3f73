"""b200_ctx_kernel_launches against the kernels CUDA itself records: over each window, the counter's increase equals the number of the library's kernel
records torch.profiler (CUDA activity, CUPTI) sees.  The windows cover the pictures whose launch counts depend on the data: an I picture without PUs
(empty lists launch nothing), B and LMCS pictures whose sparse intra lists take the one-CTA-per-block K6 kernel (the LMCS one in two passes), a 4:0:0
picture with every filter on (no chroma kernels), and the outputs that run kernels on the copy stream."""
import ctypes as C
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth
from tests.helpers import PIPELINE_KINDS, intra_dense, intra_kernel

pytestmark = pytest.mark.gpu
W, H, BD = 416, 240, 10
OUT_PYUV, OUT_8, HASH_CRC = 1, 2, 1


def counted(b200, ctx, fn):
    """(increase of the context's launch counter, kernels of the library torch.profiler recorded) while fn runs and the device drains."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        before = b200.b200_ctx_kernel_launches(ctx)
        fn()
        torch.cuda.synchronize()
        after = b200.b200_ctx_kernel_launches(ctx)
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "b200::" in e.name]
    assert kernels, "torch.profiler recorded no kernel of the library: the count cannot be checked"
    return after - before, len(kernels)


def context(b200, g):
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    for k in range(4):
        planes = synth.noise_planes(np.random.default_rng(k), g.width, g.height, g.bitDepth)
        vvdec_b200.check(b200.b200_ctx_load_slot(ctx, k, abi.plane_ptrs(planes)))
    return ctx


def picture(b200, ctx, pic):
    """upload, run, wait; returns the handle"""
    h = b200.b200_pic_upload(ctx, C.byref(pic["struct"]))
    assert h >= 0, b200.b200_last_error()
    vvdec_b200.check(b200.b200_pic_run(ctx, h))
    vvdec_b200.check(b200.b200_wait_picture(ctx, h, None, 0))
    return h


def test_i_picture_without_pus(b200):
    g = abi.make_geom(W, H, BD)
    pic = synth.gen_picture(np.random.default_rng(1), W, H, BD, dst_slot=4, **PIPELINE_KINDS["I"])
    assert len(pic["pus"]) == 0 and pic["struct"].numIntraTus
    ctx = context(b200, g)
    try:
        with intra_kernel("auto"):
            handle = []
            n, want = counted(b200, ctx, lambda: handle.append(b200.b200_pic_upload(ctx, C.byref(pic["struct"]))))
            assert handle[0] >= 0, b200.b200_last_error()
            assert n == want, f"upload: counted {n}, profiler {want}"
            n, want = counted(b200, ctx, lambda: vvdec_b200.check(b200.b200_pic_run(ctx, handle[0])))
            assert n == want, f"run: counted {n}, profiler {want}"
    finally:
        b200.b200_ctx_destroy(ctx)


@pytest.mark.parametrize("kind", ["B", "L"])
def test_sparse_intra_list(b200, kind):
    """B: the sparse intra list of a B picture; L: the same with LMCS chroma scaling, so K6 runs in two passes around the VPDU scales."""
    g = abi.make_geom(W, H, BD)
    pic = synth.gen_picture(np.random.default_rng(2), W, H, BD, dst_slot=4, **PIPELINE_KINDS[kind])
    ni = pic["struct"].numIntraTus
    assert ni and not intra_dense(g, ni) and len(pic["pus"])
    assert kind != "L" or pic["lmcs"]["struct"].chromaAdj
    ctx = context(b200, g)
    try:
        with intra_kernel("auto"):
            n, want = counted(b200, ctx, lambda: picture(b200, ctx, pic))
        assert n == want, f"{kind}: counted {n}, profiler {want}"
    finally:
        b200.b200_ctx_destroy(ctx)


def test_yuv400_with_every_filter(b200):
    g = abi.make_geom(W, H, BD, chroma_format=0, ctu=128, strides=(W, 0, 0))
    rng = np.random.default_rng(3)
    pic = synth.gen_picture(rng, W, H, BD, dst_slot=4, inter=False, tu_kw=dict(p_cbf=0.0))
    st = pic["struct"]
    assert st.flags == abi.PIC_DEBLOCK | abi.PIC_SAO | abi.PIC_ALF and st.numPus == 0 and st.numTus == 0
    given = synth.noise_planes(rng, W, H, BD, chroma=False)
    pic["given"] = given; st.given[0] = given[0].ctypes.data
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, -1))
    try:
        n, want = counted(b200, ctx, lambda: picture(b200, ctx, pic))
        assert n == want, f"4:0:0: counted {n}, profiler {want}"
    finally:
        b200.b200_ctx_destroy(ctx)


def test_outputs(b200):
    g = abi.make_geom(W, H, BD)
    rng = np.random.default_rng(4)
    pic = synth.gen_picture(rng, W, H, BD, dst_slot=4)
    ctx = context(b200, g)
    tabs = synth.gen_film_grain_tables(rng, H)
    fg = abi.FilmGrain()
    fg.pattern, fg.sLUT, fg.pLUT, fg.lineSeeds = (t.ctypes.data for t in tabs)
    fg.scaleShift = 9
    for c in range(3): fg.compPresent[c] = 1
    try:
        picture(b200, ctx, pic)
        for name, fmt in (("fmt", OUT_PYUV), ("grain", OUT_8), ("hash", HASH_CRC)):
            if name == "hash":
                dst = np.zeros(12, np.uint8)
                call = lambda: b200.b200_frame_hash_async(ctx, 4, HASH_CRC, dst.ctypes.data)
            else:
                dst = [np.zeros(b200.b200_frame_bytes(C.byref(g), fmt, c), np.uint8) for c in range(3)]
                ptrs = (C.c_void_p * 3)(*[d.ctypes.data for d in dst])
                call = (lambda: b200.b200_get_frame_fmt_async(ctx, 4, fmt, ptrs)) if name == "fmt" else (lambda: b200.b200_get_frame_grain_async(ctx, 4, fmt, ptrs, C.byref(fg)))
            t = []
            n, want = counted(b200, ctx, lambda: t.append(call()))
            assert t[0] >= 0, b200.b200_last_error()
            vvdec_b200.check(b200.b200_frame_wait(ctx, t[0]))
            assert n == want, f"{name}: counted {n}, profiler {want}"
    finally:
        b200.b200_ctx_destroy(ctx)
