"""K3 parity on the GPU: CUDA deblocking (through the C ABI) vs the pinned oracle, bit-exact, on random pictures and on every case of the designed
sweep (synth.lf_sweep); and the wrapper's refusals, each next to the same call with the offending field fixed."""
import ctypes as C
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth
from tests.helpers import lf_args, lf_oracle, lf_mismatch
from tests.test_k3_oracle_vs_ref import _picture_case
from tests.test_k3_cases_cpu import REFUSALS, refusal_base, refusal_variant

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed,W,H,bd,ctu,nsl,ladf", [(1, 256, 128, 10, 128, 1, 0), (2, 416, 240, 10, 64, 2, 1), (3, 200, 136, 8, 32, 3, 0),
                                                     (4, 1920, 1080, 10, 128, 1, 0), (5, 384, 256, 12, 128, 1, 1),
                                                     (6, 3840, 2160, 10, 128, 1, 0)])
@pytest.mark.parametrize("dirs", [1, 2, 3])
def test_deblock_gpu_vs_oracle(b200, oracle, seed, W, H, bd, ctu, nsl, ladf, dirs):
    if W >= 1920 and dirs != 3:
        pytest.skip("large pictures: full V+H only")
    rng = np.random.default_rng(seed)
    cus, lfV, lfH, planes, sl, ctu_slice, seq = _picture_case(rng, W, H, bd, ctu, nsl, ladf)
    g = abi.make_geom(W, H, bd, ctu=ctu)
    a = [p.copy() for p in planes]; b = [p.copy() for p in planes]
    oracle.orc_lf_deblock(C.byref(g), abi.plane_ptrs(a), lfV.ctypes.data, lfH.ctypes.data, ctu_slice.ctypes.data,
                          sl.ctypes.data, C.addressof(seq), dirs)
    vvdec_b200.check(b200.b200_lf_deblock(C.byref(g), abi.plane_ptrs(b), lfV.ctypes.data, lfH.ctypes.data,
                                          ctu_slice.ctypes.data, sl.ctypes.data, nsl, C.addressof(seq), dirs))
    for c in range(3):
        assert np.array_equal(a[c], b[c]), f"plane {c}: {np.argwhere(a[c] != b[c])[:8]}"
    assert not np.array_equal(a[0], planes[0])


def _run(b200, case, dirs, planes=None, nsl=None):
    out = [None if p is None else p.copy() for p in (planes or case["planes"])]
    rc = b200.b200_lf_deblock(*lf_args(case, out), len(case["slices"]) if nsl is None else nsl, C.addressof(case["seq"]), dirs)
    return rc, out


_SMALL = [n for n in synth.LF_SWEEP_CASES if synth.lf_sweep(n)["W"] * synth.lf_sweep(n)["H"] <= 1 << 20]


@pytest.mark.parametrize("name,dirs", [(n, d) for n in synth.LF_SWEEP_CASES for d in ((1, 2, 3) if n in _SMALL else (3,))])
def test_deblock_designed_sweep(b200, oracle, name, dirs):
    """Every case of the designed sweep: each decision with its thresholds on both sides, every long pair, chroma CTB forms at CTU 32 / 64 / 128, QP
    and offset extremes at 8 / 9 / 10 / 12 bit, LADF with 5 intervals, clipping at 0 and pmax, legal grids at minimum spacing with crossing edges,
    CTU rows and partial CTUs, 64 slices, 4:0:0, padded and odd strides and a 4K picture.  The planes (stride padding included) equal the oracle's; a
    failure names the case, plane, position and the classified decision of the segment that writes it."""
    case = synth.lf_sweep(name)
    want = lf_oracle(oracle, case, dirs)
    rc, got = _run(b200, case, dirs)
    vvdec_b200.check(rc)
    msg = lf_mismatch(oracle, case, got, want, dirs)
    assert msg is None, msg


@pytest.mark.parametrize("what,bad,fixed,grid", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_deblock_refusals(b200, oracle, what, bad, fixed, grid):
    """Each rule of b200_lf_deblock's host checks, alone, makes it return B200_ERR_PARAM with an error message and the host planes untouched; the same
    call with the offending field fixed is accepted and equals the oracle.  The refused calls never reach the device or the oracle."""
    ok = refusal_variant(fixed)
    rc, got = _run(b200, ok, ok["dirs"])
    assert rc == 0, (what, b200.b200_last_error())
    msg = lf_mismatch(oracle, ok, got, lf_oracle(oracle, ok, ok["dirs"]), ok["dirs"])
    assert msg is None, msg
    k = refusal_variant(bad)
    planes = [None if p is None else np.full_like(p, -5) for p in k["planes"]]
    rc, got = _run(b200, k, k["dirs"], planes=planes)
    assert rc == -2, (what, rc)
    assert b"b200_lf_deblock" in b200.b200_last_error(), what
    assert all(p is None or (p == -5).all() for p in got), what
