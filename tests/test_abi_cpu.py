"""CPU-side checks of the boundary: the library loads without a GPU and exports every symbol of include/vvdec_b200.h."""
import os, re, ctypes as C
import numpy as np
import vvdec_b200
from vvdec_b200 import abi, bindings, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "vvdec_b200.h")).read()
    declared = set(re.findall(r"B200_API\s+[\w\s\*]+?\b(b200_\w+)\s*\(", hdr))
    assert declared, "no B200_API declarations found"
    lib = C.CDLL(vvdec_b200.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert declared == set(bindings.EXPORTS), declared ^ set(bindings.EXPORTS)


def test_struct_sizes_match_header():
    assert C.sizeof(abi.Tu) == 32 and abi.TU_DTYPE.itemsize == 32
    assert C.sizeof(abi.Geom) == 32


def test_no_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        return
    lib = vvdec_b200.lib()
    g = abi.make_geom(64, 64, 10)
    planes = [np.zeros((64, 64), np.int16), np.zeros((32, 32), np.int16), np.zeros((32, 32), np.int16)]
    rc = lib.b200_k1_residual(C.byref(g), abi.plane_ptrs(planes), None, 0, None, 0, None, 0, 0)
    assert rc == -3 and b"no CPU fallback" in lib.b200_last_error()


def test_records_are_refused_before_device_work():
    """b200_mc_predict and b200_k1_residual check every record on the host before they look for a device: one bad PU / TU is refused with
    B200_ERR_PARAM on any machine, naming the record, and the same call with the record fixed is not."""
    from tests.helpers import mc_dst, ref_ptrs
    refusal = synth.library_refusal
    g = abi.make_geom(64, 64, 10)
    refs = [synth.noise_planes(np.random.default_rng(1), 64, 64, 10)]
    pus = np.array([synth._mc_pu(0, 0, 16, 16, (0, -1)), synth._mc_pu(16, 0, 16, 16, (0, -1))], synth.PU_DTYPE)
    dst = mc_dst(g)                                   # alive while the library writes it (on a GPU)
    mc = lambda: refusal("b200_mc_predict", C.byref(g), abi.plane_ptrs(dst), ref_ptrs(refs), 1, pus.ctypes.data, len(pus), None, 0)
    assert mc() is None
    pus["refSlot"][1] = (1, -1)
    assert "b200_mc_predict: PU 1: invalid reference slots" in mc()
    tus = np.zeros(1, abi.TU_DTYPE)
    tus["log2w"], tus["log2h"], tus["inBits"] = 2, 2, 16
    coefs = np.zeros(1, np.int16)
    k1 = lambda: refusal("b200_k1_residual", C.byref(g), abi.plane_ptrs(dst), tus.ctypes.data, 1, coefs.ctypes.data, 1, None, 0, 0)
    assert k1() is None
    tus["log2w"] = 7
    assert "b200_k1_residual: TU record 0" in k1()


def test_partition_tiles_picture_exactly():
    rng = np.random.default_rng(0)
    for (W, H) in [(416, 240), (1920, 1080), (136, 72)]:
        cus = synth.partition(rng, W, H)
        cover = np.zeros((H, W), np.int32)
        for x, y, w, h in cus:
            assert x + w <= W and y + h <= H
            cover[y:y + h, x:x + w] += 1
        assert (cover == 1).all()
