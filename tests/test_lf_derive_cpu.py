"""Edge grids derived from CU / TU records (B200_PIC_DERIVE_LF, vvdec_b200/csrc/lf_derive.cuh) against the reference's own derivation.

  * Everywhere: the derivation compiled for the host from the same header (tests/lf_derive_host.cpp, built here with the host C++ compiler) on the records of
    tests/golden/lf_derive_pictures.npz (tools/make_golden.py: seam pictures as the drop-in class flattens them with the derivation on) gives the reference's
    grids of those pictures byte for byte; a slice with deblocking disabled ends its CTUs; b200_lf_derive refuses bad records before it looks for a device.
  * Where oracle/_ref holds a build of the current glue: the drop-in class flattens each seam picture (oracle/ref_seam.h) and every picture of the stream cases
    and seeded fuzz streams twice without a device — as it always does (LoopFilter::calcFilterStrengthsCTU, then flattenLfCtu), and with the derivation switched on
    (B200_LF_DERIVE=1), where it emits the records and runs lf_derive_serial — and both lfV / lfH rasters must be byte-identical."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import numpy as np
import pytest
from tests import helpers
from vvdec_b200 import abi

ref = helpers.load_ref()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lf_derive_pictures.npz")


def built_with_derivation(path):
    """The glue compiled into this oracle/_ref library reads B200_LF_DERIVE, i.e. it was built from glue that has the device edge derivation: oracle/_ref is
    built where the reference sources are, so elsewhere it may be an older build."""
    if not os.path.exists(path): return False
    with open(path, "rb") as f: return b"B200_LF_DERIVE" in f.read()


needs_glue = pytest.mark.skipif(ref is None or not hasattr(ref, "ref_seam_create") or not built_with_derivation(helpers.REF_SO),
                                reason="oracle/_ref is not built, or was built from a glue without the device edge derivation (build() rebuilds it where the reference sources are)")

ALL_TOOLS = helpers.SEAM_INTER_TOOLS | helpers.SEAM_RESI_TOOLS | helpers.SEAM_INTRA_TOOLS | helpers.SEAM_FILTERS
CASES = {
    "B_mixed": dict(),                                                          # affine, SbTMVP, GEO, CIIP, SBT, JCCR, BDPCM among 15 % intra CUs
    "B_intra_heavy": dict(intra=45, skip=5),
    "B_affine_heavy": dict(affine=60, intra=5),
    "I_picture": dict(slice_type=2),
    "P_picture": dict(slice_type=1),
    "B_isp": dict(isp=60, intra=40),
    "I_isp": dict(isp=60, slice_type=2),
    "B_3slices": dict(slices=3),
    "P_5slices": dict(slices=5, slice_type=1),
    "B_5slices_no_lf_across_ctu64": dict(slices=5, ctu=64, lf_across_slices=False),
    "I_6slices_no_lf_across_ctu64": dict(slices=6, ctu=64, lf_across_slices=False, slice_type=2),
    "B_local_dual_tree_isp": dict(tools=ALL_TOOLS | helpers.SEAM["LOCAL_DUAL_TREE"], isp=40),
    "I_local_dual_tree": dict(tools=ALL_TOOLS | helpers.SEAM["LOCAL_DUAL_TREE"], slice_type=2),
    "B_ctu64": dict(ctu=64),
    "B_ctu32_8bit": dict(ctu=32, bd=8),
    "B_lmcs": dict(lmcs=True),
}
SIZES = {"416x240": (416, 240), "200x136": (200, 136)}                          # 200x136: not a multiple of any CTU size


def flatten_grids(case, derive):
    """(lfV, lfH, picture struct) of one dry run of the drop-in class, with the device derivation switched on or off."""
    old = os.environ.get("B200_LF_DERIVE")
    os.environ["B200_LF_DERIVE"] = "1" if derive else "0"
    try:
        h = case.build(); flat = abi.Picture(); col = np.zeros(ref.ref_seam_col_motion_bytes(h), np.uint8)
        secs = ref.ref_seam_run_b200(h, 0, 1, None, col.ctypes.data, len(col), C.byref(flat))
        ref.ref_seam_destroy(h)
    finally:
        if old is None: del os.environ["B200_LF_DERIVE"]
        else: os.environ["B200_LF_DERIVE"] = old
    assert secs >= 0, f"DecLibReconB200 refused the picture ({secs})"
    n4 = (case.g.width >> 2) * (case.g.height >> 2)
    grids = []
    for p in (flat.lfV, flat.lfH):
        assert p, "no deblocking grid in the flattened picture"
        grids.append(np.frombuffer((C.c_uint8 * (6 * n4)).from_address(p), abi.LF_PARAM_DTYPE).copy())
    return grids[0], grids[1], flat


def first_difference(want, got, W4):
    """The first entry (raster order) whose fields differ, named by field: bs per component, qp[3], sideMaxFiltLength, flags."""
    for i in range(len(want)):
        a, b = want[i], got[i]
        if a.tobytes() == b.tobytes(): continue
        diffs = []
        for c, name in enumerate(("Y", "Cb", "Cr")):
            if (int(a["bs"]) >> 2 * c) & 3 != (int(b["bs"]) >> 2 * c) & 3: diffs.append(f"bs[{name}] {(int(a['bs']) >> 2 * c) & 3} != {(int(b['bs']) >> 2 * c) & 3}")
        if int(a["bs"]) >> 6 != int(b["bs"]) >> 6: diffs.append(f"bs transient bits {int(a['bs']) >> 6} != {int(b['bs']) >> 6}")
        if list(a["qp"]) != list(b["qp"]): diffs.append(f"qp {list(a['qp'])} != {list(b['qp'])}")
        for f in ("sideMaxFiltLength", "flags"):
            if a[f] != b[f]: diffs.append(f"{f} {int(a[f]):#x} != {int(b[f]):#x}")
        return f"luma ({4 * (i % W4)}, {4 * (i // W4)}): " + "; ".join(diffs)
    return None


def check_case(seed, W, H, **kw):
    case = helpers.SeamCase(ref, np.random.default_rng(seed), W, H, **kw)
    wantV, wantH, _ = flatten_grids(case, False)
    gotV, gotH, flat = flatten_grids(case, True)
    assert flat.lfCus and flat.numLfCus > 0 and flat.lfTus and flat.numLfTus >= flat.numLfCus, "no CU / TU records in the derived picture"
    W4 = W >> 2
    for name, want, got in (("lfV", wantV, gotV), ("lfH", wantH, gotH)):
        assert want.tobytes() == got.tobytes(), f"{name}: {first_difference(want, got, W4)}"
    return wantV, wantH


@needs_glue
@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_derived_grids_equal_calc_filter_strengths(name, seed, size):
    check_case(seed, *SIZES[size], **CASES[name])


@needs_glue
def test_the_cases_reach_every_edge_kind():
    """The designed cases put strong (2), normal (1) and zero luma Bs, transform and sub-block edges and long luma filters into the grids."""
    bs, lens = set(), set()
    for name in ("B_mixed", "I_picture", "B_affine_heavy"):
        V, Hh = check_case(5, 416, 240, **CASES[name])
        for g in (V, Hh):
            bs |= set(int(b) & 3 for b in g["bs"])
            lens |= set(int(s) & 0x77 for s in g["sideMaxFiltLength"])
    assert bs >= {0, 1, 2}, bs
    assert {0x33, 0x77, 0x11, 0x22} & lens, lens


@needs_glue
def test_larger_picture_on_a_thread_pool():
    """Flatten rows run on the pool in any order: the records are joined in CTU order all the same."""
    case = helpers.SeamCase(ref, np.random.default_rng(31), 832, 480)
    os.environ["B200_LF_DERIVE"] = "1"
    try:
        h = case.build(); flat = abi.Picture(); col = np.zeros(ref.ref_seam_col_motion_bytes(h), np.uint8)
        assert ref.ref_seam_run_b200(h, 4, 1, None, col.ctypes.data, len(col), C.byref(flat)) >= 0
        ref.ref_seam_destroy(h)
        n4 = (832 >> 2) * (480 >> 2)
        got = [np.frombuffer((C.c_uint8 * (6 * n4)).from_address(p), np.uint8).copy() for p in (flat.lfV, flat.lfH)]
    finally:
        del os.environ["B200_LF_DERIVE"]
    wantV, wantH, _ = flatten_grids(case, False)
    assert got[0].tobytes() == wantV.tobytes() and got[1].tobytes() == wantH.tobytes()


def records_of(flat, g):
    """Copies of a derived picture's records, as the arguments of b200_lf_derive take them."""
    nCtu = ((g.width + g.ctuSize - 1) // g.ctuSize) * ((g.height + g.ctuSize - 1) // g.ctuSize)
    cp = lambda p, n, dt: np.frombuffer((C.c_uint8 * (n * np.dtype(dt).itemsize)).from_address(p), dt).copy() if n else np.zeros(0, dt)
    return dict(cus=cp(flat.lfCus, flat.numLfCus, abi.LF_CU_DTYPE), tus=cp(flat.lfTus, flat.numLfTus, abi.LF_TU_DTYPE),
                ctuCus=cp(flat.lfCtuCus, nCtu + 1, np.uint32), pus=cp(flat.pus, flat.numPus, np.dtype((np.void, 64))),
                slices=cp(flat.lfSlices, flat.numLfSlices, np.dtype((np.void, 8))), sliceB=cp(flat.lfSliceB, flat.numLfSlices, np.uint8))


def lf_derive(fn, g, r):
    """fn: b200_lf_derive, or lf_derive_host (same arguments).  Returns (rc, lfV, lfH)."""
    n4 = (g.width >> 2) * (g.height >> 2)
    V, H = np.zeros(n4, abi.LF_PARAM_DTYPE), np.zeros(n4, abi.LF_PARAM_DTYPE)
    rc = fn(C.byref(g), r["cus"].ctypes.data, len(r["cus"]), r["tus"].ctypes.data, len(r["tus"]), r["ctuCus"].ctypes.data,
                            r["pus"].ctypes.data if len(r["pus"]) else None, len(r["pus"]), r["slices"].ctypes.data, r["sliceB"].ctypes.data, len(r["slices"]),
                            V.ctypes.data, H.ctypes.data)
    return rc, V, H


# ---- the golden pictures: no oracle/_ref needed ----
def golden():
    z = np.load(GOLDEN)
    out = []
    for k, name in enumerate(z["names"]):
        gv = z[f"{k}_geom"]
        g = abi.make_geom(int(gv[0]), int(gv[1]), int(gv[3]), int(gv[2]), int(gv[4]))
        r = {f: np.ascontiguousarray(z[f"{k}_{f}"]) for f in ("cus", "tus", "ctuCus", "pus", "slices", "sliceB")}
        out.append((str(name), g, r, z[f"{k}_lfV"], z[f"{k}_lfH"]))
    return out


GOLDEN_NAMES = [c[0] for c in golden()]


@pytest.fixture(scope="module")
def host():
    """tests/lf_derive_host.cpp built with the host C++ compiler into a temporary directory."""
    cxx = shutil.which(os.environ.get("CXX", "g++")) or shutil.which("g++") or shutil.which("c++")
    assert cxx, "no host C++ compiler"
    d = tempfile.mkdtemp(prefix="lf_derive_host_")
    so = os.path.join(d, "lf_derive_host.so")
    subprocess.check_call([cxx, "-std=c++14", "-O2", "-w", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "lf_derive_host.cpp")])
    lib = C.CDLL(so)
    lib.lf_derive_host.argtypes = [C.POINTER(abi.Geom), C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t,
                                   C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    yield lib.lf_derive_host
    shutil.rmtree(d, ignore_errors=True)


def with_disabled_slice(g, r, lfV, lfH, disabled):
    """Records with slice `disabled` switched to deblocking off, and the grids the reference gives then: calcFilterStrengthsCTU returns for the rest of a
    CTU at the first CU of such a slice (LoopFilter.cpp:364-369) and entries no CU writes stay zero; a CU writes only entries of its own block, so they are the
    grids with every later CU of such a CTU cleared.  Returns (records, lfV, lfH, number of CUs cut)."""
    r = {k: v.copy() for k, v in r.items()}; V, H = lfV.copy(), lfH.copy()
    r["slices"].view(np.uint8).reshape(-1, 8)[disabled, 6] = 1                 # b200_lf_slice::disable
    W4, cut = g.width >> 2, 0
    for a in range(len(r["ctuCus"]) - 1):
        stop = False
        for i in range(int(r["ctuCus"][a]), int(r["ctuCus"][a + 1])):
            cu = r["cus"][i]
            stop = stop or int(cu["slice"]) == disabled
            if stop:
                assert cu["chType"] == 0
                x4, y4, w4, h4 = cu["x"] >> 2, cu["y"] >> 2, cu["w"] >> 2, cu["h"] >> 2
                for want in (V, H): want.reshape(-1, W4)[y4:y4 + h4, x4:x4 + w4] = np.zeros((), abi.LF_PARAM_DTYPE)
                cut += 1
    return r, V, H, cut


def check_grids(g, want, got):
    W4 = g.width >> 2
    for k, a, b in (("lfV", want[0], got[0]), ("lfH", want[1], got[1])):
        assert a.tobytes() == b.tobytes(), f"{k}: {first_difference(a, b, W4)}"


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_golden_records_give_the_reference_grids(host, name):
    g, r, wantV, wantH = next((c[1], c[2], c[3], c[4]) for c in golden() if c[0] == name)
    rc, V, H = lf_derive(host, g, r)
    assert rc == 0
    check_grids(g, (wantV, wantH), (V, H))


@pytest.mark.parametrize("disabled", [1, 2])
def test_slice_with_deblocking_disabled_ends_its_ctus(host, disabled):
    """Raster slices that start inside CTU rows (the golden three-slice picture, CTU 128)."""
    g, r, wantV, wantH = next((c[1], c[2], c[3], c[4]) for c in golden() if c[0].startswith("B_3slices"))
    r, wantV, wantH, cut = with_disabled_slice(g, r, wantV, wantH, disabled)
    assert cut > 0
    rc, V, H = lf_derive(host, g, r)
    assert rc == 0
    check_grids(g, (wantV, wantH), (V, H))


def test_golden_pictures_reach_every_edge_kind():
    """Strong (2), normal (1) and zero luma Bs, short and long luma filters, chroma-tree, ISP, affine, GEO, CIIP and BDPCM CUs.  (The seam generator draws no
    SbTMVP CUs; the stream cases, which do, run through test_stream_pictures_derive_the_same_grids.)"""
    bs, lens, flags, ch = set(), set(), 0, set()
    for _, g, r, V, H in golden():
        for grid in (V, H):
            bs |= set(int(b) & 3 for b in grid["bs"]); lens |= set(int(s) & 0x77 for s in grid["sideMaxFiltLength"])
        for f in r["cus"]["flags"]: flags |= int(f)
        ch |= set(int(c) for c in r["cus"]["chType"])
    assert bs >= {0, 1, 2}, bs
    assert {0x11, 0x33, 0x77} <= lens, lens
    for f in (abi.LF_CU_ISP, abi.LF_CU_AFFINE, abi.LF_CU_GEO, abi.LF_CU_CIIP, abi.LF_CU_SEP_TREE, abi.LF_CU_BDPCM_Y):
        assert flags & f, f
    assert ch == {0, 1}


def test_b200_lf_derive_refuses_bad_records_before_any_device_work():
    """The kernel-level derivation checks every CU / TU record with the picture path's rule (rules.cuh: lf_cu_problem) before it looks for a device."""
    import vvdec_b200
    lib = vvdec_b200.lib()
    g, good = next((c[1], c[2]) for c in golden() if c[0].startswith("B_5slices"))
    rc, _, _ = lf_derive(lib.b200_lf_derive, g, good)
    assert rc in (0, -3), lib.b200_last_error()                                     # valid records: derived (GPU) or B200_ERR_NO_DEVICE (no GPU)
    cu0 = int(good["ctuCus"][1])                                                    # the first CU record of the second CTU
    bad_cases = {
        "CU outside its CTU": lambda r: r["cus"][cu0].__setitem__("x", 0),
        "CU outside the picture": lambda r: r["cus"][-1].__setitem__("w", 255),
        "slice index": lambda r: r["cus"][0].__setitem__("slice", len(r["slices"])),
        "TU records past numLfTus": lambda r: r["cus"][-1].__setitem__("firstTu", len(r["tus"])),
        "no TU": lambda r: r["cus"][0].__setitem__("numTus", 0),
        "TU outside the CTU": lambda r: r["tus"][int(r["cus"][cu0]["firstTu"])].__setitem__("x", 0),
        "undefined flag": lambda r: r["cus"][0].__setitem__("flags", 0x800),
        "chroma channel type": lambda r: r["cus"][0].__setitem__("chType", 2),
        "CTU ranges": lambda r: r["ctuCus"].__setitem__(-1, len(r["cus"]) + 1),
    }
    for name, spoil in bad_cases.items():
        r = {k: v.copy() for k, v in good.items()}
        spoil(r)
        rc, V, H = lf_derive(lib.b200_lf_derive, g, r)
        assert rc == -2, (name, rc)
        assert not V.view(np.uint8).any() and not H.view(np.uint8).any(), name


# ---- bitstreams: every picture of the stream cases and of seeded fuzz streams, as the swapped decoder hands them over ----
STREAMS = [f"{n}-s1" for n in __import__("tests.test_stream_cpu", fromlist=["CASES"]).CASES] + [f"fuzz{s}" for s in range(7000, 7040)]


def decode_records(aus, samples, derive):
    from tests import stream_util as su
    old = os.environ.get("B200_LF_DERIVE")
    os.environ["B200_LF_DERIVE"] = "1" if derive else "0"
    try:
        records = []
        frames, _ = su.decode_swapped_cpu(aus, helpers.load_oracle(), keep=records, frame_samples=samples)
    finally:
        if old is None: del os.environ["B200_LF_DERIVE"]
        else: os.environ["B200_LF_DERIVE"] = old
    return frames, records


@needs_glue
@pytest.mark.parametrize("name", STREAMS)
def test_stream_pictures_derive_the_same_grids(name):
    """The swapped decoder (glue host stages + the oracle chain in place of the device) with the derivation on: every picture's grids equal the ones
    calcFilterStrengthsCTU gives, and the frames equal the stock decoder's."""
    from oracle import vvc_stream as vs
    from tests import stream_util as su
    from tests.test_stream_cpu import _diff
    if not (vs.available() and built_with_derivation(vs.SWAP_SO)): pytest.skip("oracle/_ref/libvvdec_swapped.so is not built from the current glue")
    aus, pics, samples, _ = su.corpus_stream(name)
    stock = vs.decode(vs.REF_SO, aus, frame_samples=samples)
    _, want = decode_records(aus, samples, False)
    frames, got = decode_records(aus, samples, True)
    assert len(want) == len(got) == len(pics)
    for i, (a, b) in enumerate(zip(want, got)):
        W4 = a["geom"].width >> 2
        assert ("lfV" in a["pic"]) == ("lfV" in b["pic"]), f"picture {i}: deblocking on in one run only"
        for k in ("lfV", "lfH") if "lfV" in a["pic"] else ():
            assert a["pic"][k].tobytes() == b["pic"][k].tobytes(), f"picture {i} (POC {a['poc']}) {k}: {first_difference(a['pic'][k].view(abi.LF_PARAM_DTYPE), b['pic'][k].view(abi.LF_PARAM_DTYPE), W4)}"
    assert _diff(frames, stock) == [0] * len(stock)
