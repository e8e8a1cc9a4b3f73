"""Test helpers: load the oracle (C restatement) and, when built, the reference shim."""
import contextlib, functools, os, subprocess, ctypes as C
import numpy as np
from vvdec_b200 import abi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "oracle", "liboracle.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libvvdec_ref.so")

i16p = np.ctypeslib.ndpointer(np.int16, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i16p_off = C.c_void_p   # pointer into the middle of a buffer


class Cclm(C.Structure):
    """orc_cclm (oracle/vvc_oracle.h): what the oracle derives for one CCLM record."""
    _fields_ = [(n, C.c_int32) for n in ("a", "b", "shift", "minL", "maxL", "minC", "maxC", "cntT", "cntL", "normDiff", "clamped")] + \
               [("selL", C.c_int32 * 4), ("selC", C.c_int32 * 4), ("blkMin", C.c_int32), ("blkMax", C.c_int32)]


def cclm_params(oracle, g, planes, rec):
    """orc_cclm_params of one record (a numpy INTRA_TU_DTYPE scalar or row) over `planes`."""
    r = np.array(rec, abi.INTRA_TU_DTYPE).reshape(1)
    out = Cclm()
    oracle.orc_cclm_params(C.byref(g), abi.plane_ptrs(planes), r.ctypes.data, C.byref(out))
    return out


class IntraProbe(C.Structure):
    """orc_intra_trace (oracle/vvc_oracle.h): what the oracle's prediction of one regular intra record went through."""
    _fields_ = [(n, C.c_int32) for n in ("substMin", "substMax", "cubicMin", "cubicMax", "pdpcMin", "pdpcMax", "mipMin", "mipMax", "recoMin", "recoMax",
                                         "predMin", "predMax", "filtered", "interp", "mipSizeId", "mipInputOffset", "mipInput0")]


def intra_probes(oracle, g, planes, recs, resi=None):
    """orc_intra_probe of every record of a list, run in list order over copies of `planes` (as orc_intra_reconstruct runs it with `resi`)."""
    work = [None if p is None else p.copy() for p in planes]
    out = []
    for r in recs:
        one = np.array(r, abi.INTRA_TU_DTYPE).reshape(1)
        pr = IntraProbe()
        oracle.orc_intra_probe(C.byref(g), abi.plane_ptrs(work), None if resi is None else abi.plane_ptrs(resi), one.ctypes.data, C.byref(pr))
        out.append(pr)
    return out


def load_oracle():
    srcs = [os.path.join(ROOT, "oracle", f) for f in os.listdir(os.path.join(ROOT, "oracle")) if f.endswith((".c", ".h"))]
    if not os.path.exists(ORACLE_SO) or any(os.path.getmtime(s) > os.path.getmtime(ORACLE_SO) for s in srcs):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s"])
    lib = C.CDLL(ORACLE_SO)
    lib.orc_dequant.argtypes = [C.c_int] * 4 + [C.c_void_p, i16p, C.c_size_t, i32p, C.c_int, C.c_int, C.c_int32]
    lib.orc_inv_lfnst.argtypes = [i32p, i32p, C.c_uint, C.c_uint, C.c_uint, C.c_int]
    lib.orc_inv_1d.argtypes = [C.c_int, C.c_int, i32p, i32p] + [C.c_int] * 5 + [C.c_int32, C.c_int32]
    lib.orc_cpy_resi_clip.argtypes = [i32p, i16p, C.c_ssize_t, C.c_uint, C.c_uint] + [C.c_int32] * 4
    lib.orc_tu_residual.argtypes = [C.POINTER(abi.Tu), C.c_int, i16p, C.c_void_p, i16p, C.c_ssize_t]
    lib.orc_k1_residual.argtypes = [C.POINTER(abi.Geom), C.POINTER(C.POINTER(C.c_int16)), C.c_void_p, C.c_size_t,
                                    i16p, C.c_void_p, C.c_int]
    PL = C.POINTER(C.POINTER(C.c_int16))
    lib.orc_lf_pel_filter_luma.argtypes = [i16p_off, C.c_ssize_t, C.c_ssize_t] + [C.c_int] * 6
    lib.orc_lf_filtering_pq.argtypes = [i16p_off, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_int]
    lib.orc_lf_deblock.argtypes = [C.POINTER(abi.Geom), PL, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    V = C.c_void_p
    lib.orc_sao_offset_block.argtypes = [C.c_int, C.c_int, V, V, V, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_uint, C.c_int, V, C.c_int, V]
    lib.orc_sao_picture.argtypes = [C.POINTER(abi.Geom), PL, PL, V, V]
    lib.orc_alf_classify.argtypes = [V, V, C.c_ssize_t] + [C.c_int] * 7
    lib.orc_alf_filter_blk.argtypes = [C.c_int, V, V, C.c_ssize_t, V, C.c_ssize_t] + [C.c_int] * 4 + [V, V] + [C.c_int] * 3
    lib.orc_alf_ccalf_blk.argtypes = [V, C.c_ssize_t, V, C.c_ssize_t] + [C.c_int] * 4 + [V] + [C.c_int] * 3
    lib.orc_alf_picture.argtypes = [C.POINTER(abi.Geom), PL, PL, V, C.POINTER(abi.AlfTables)]
    lib.orc_mc_predict.argtypes = [C.POINTER(abi.Geom), PL, C.POINTER(C.c_void_p), V, C.c_size_t, V]
    lib.orc_mc_predict_wp.argtypes = [C.POINTER(abi.Geom), PL, C.POINTER(C.c_void_p), V, C.c_size_t, V, V]
    LP = C.POINTER(abi.Lmcs)
    lib.orc_lmcs_fwd_block.argtypes = [V, C.c_ssize_t, C.c_int, C.c_int, C.c_int, LP]
    lib.orc_lmcs_fwd_pus.argtypes = [C.POINTER(abi.Geom), i16p, V, C.c_size_t, LP]
    lib.orc_lmcs_vpdu_scale.argtypes = [C.POINTER(abi.Geom), i16p, LP, C.POINTER(abi.LmcsVpdu)]
    lib.orc_lmcs_scale_resi.argtypes = [C.c_int] * 3
    lib.orc_k1_residual_lmcs.argtypes = [C.POINTER(abi.Geom), PL, V, C.c_size_t, i16p, V, LP]
    lib.orc_lmcs_inv_plane.argtypes = [C.POINTER(abi.Geom), i16p, LP]
    lib.orc_lmcs_vpdu_scales.argtypes = [C.POINTER(abi.Geom), i16p, LP, C.c_void_p]
    lib.orc_k1_residual_sel.argtypes = [C.POINTER(abi.Geom), PL, PL, C.c_void_p, C.c_size_t, i16p, C.c_void_p, C.c_int, C.c_void_p]
    u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
    lib.orc_pack_pyuv.argtypes = [i16p, C.c_ssize_t, C.c_int, C.c_int, u8p]
    lib.orc_narrow8.argtypes = [i16p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, u8p]
    lib.orc_intra_predict.argtypes = [C.POINTER(abi.Geom), PL, C.c_void_p, C.c_size_t]
    lib.orc_intra_isp_cu.argtypes = [C.POINTER(abi.Geom), i16p, C.c_void_p] + [C.c_int] * 11 + [C.c_uint]
    lib.orc_intra_reconstruct.argtypes = [C.POINTER(abi.Geom), PL, PL, C.c_void_p, C.c_size_t]
    lib.orc_cclm_params.argtypes = [C.POINTER(abi.Geom), PL, C.c_void_p, C.POINTER(Cclm)]
    lib.orc_intra_probe.argtypes = [C.POINTER(abi.Geom), PL, PL, C.c_void_p, C.POINTER(IntraProbe)]
    lib.orc_film_grain.argtypes = [PL, C.POINTER(C.c_ssize_t), C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.orc_plane_hash.argtypes = [C.c_int, C.c_int, i16p, C.c_ssize_t, C.c_int, C.c_int, u8p]
    return lib


class RefTuSyntax(C.Structure):
    _fields_ = [(n, C.c_int32) for n in
                ["w", "h", "comp", "bitDepth", "predMode", "qp", "chromaQpAdj", "cbQpOffset", "crQpOffset",
                 "jointQpOffset", "depQuant", "mtsIdx", "lfnstIdx", "intraDirL", "intraDirC", "mipFlag", "ispMode",
                 "sbtIdx", "sbtPos", "bdpcmL", "bdpcmC", "jointCbCr", "jointCbCrSign", "maxScanPosX", "maxScanPosY",
                 "spsMTS", "spsIntraMTS", "spsInterMTS", "spsLFNST", "sepTree"]]


_ref_lib = None                                               # set once the compiled reference has been loaded (tests/conftest.py leaves without its static destructors)


def load_ref():
    global _ref_lib
    if not os.path.exists(REF_SO):
        return None
    lib = C.CDLL(REF_SO); _ref_lib = lib
    lib.ref_simd_level.restype = C.c_char_p
    lib.ref_dequant.argtypes = [C.c_int] * 5 + [i16p, C.c_size_t, i32p, C.c_int, C.c_int, C.c_int32]
    lib.ref_dequant_scaling.argtypes = [C.c_int] * 5 + [i32p, i16p, C.c_size_t, i32p, C.c_int, C.c_int, C.c_int32]
    lib.ref_inv_lfnst.argtypes = [i32p, i32p, C.c_uint, C.c_uint, C.c_uint, C.c_int]
    lib.ref_inv_1d.argtypes = [C.c_int, C.c_int, C.c_int, i32p, i32p] + [C.c_int] * 5 + [C.c_int32, C.c_int32]
    lib.ref_cpy_resi_clip.argtypes = [C.c_int, i32p, i16p, C.c_ssize_t, C.c_uint, C.c_uint] + [C.c_int32] * 4
    lib.ref_tu_case.argtypes = [C.POINTER(RefTuSyntax), i16p, i16p, i16p, C.POINTER(abi.Tu), i16p, C.POINTER(C.c_int32)]
    lib.ref_tu_case.restype = C.c_int
    PL = C.POINTER(C.POINTER(C.c_int16))
    lib.ref_lf_pel_filter_luma.argtypes = [C.c_int, i16p_off, C.c_ssize_t, C.c_ssize_t] + [C.c_int] * 6
    lib.ref_lf_filtering_pq.argtypes = [C.c_int, i16p_off, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_int]
    lib.ref_lf_deblock_picture.argtypes = [C.c_int, C.POINTER(abi.Geom), PL, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    V = C.c_void_p
    lib.ref_sao_offset_block.argtypes = [C.c_int, C.c_int, C.c_int, V, C.c_int, V, V, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_uint, C.c_int, V, C.c_int, V]
    lib.ref_sao_picture.argtypes = [C.c_int, C.POINTER(abi.Geom), PL, PL, V, V]
    lib.ref_alf_classify.argtypes = [C.c_int, V, V, C.c_ssize_t] + [C.c_int] * 9
    lib.ref_alf_filter_blk.argtypes = [C.c_int, C.c_int, V, V, C.c_ssize_t, V, C.c_ssize_t] + [C.c_int] * 6 + [V, V] + [C.c_int] * 3
    lib.ref_alf_ccalf_blk.argtypes = [C.c_int, V, C.c_ssize_t, V, C.c_ssize_t] + [C.c_int] * 6 + [V] + [C.c_int] * 3
    lib.ref_alf_picture.argtypes = [C.c_int, C.POINTER(abi.Geom), PL, PL, V, C.POINTER(abi.AlfTables)]
    lib.ref_mc_predict.argtypes = [C.c_int, C.POINTER(abi.Geom), PL, C.POINTER(C.c_void_p), V, C.c_size_t, V, C.c_size_t]
    lib.ref_mc_predict.restype = C.c_int
    lib.ref_set_wp.argtypes = [C.c_void_p]
    lib.ref_flatten_pu_case.argtypes = [C.c_int, C.POINTER(abi.Geom), C.POINTER(C.c_void_p), C.c_int, C.c_void_p, C.c_int, PL, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    lib.ref_write_component.argtypes = [i16p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS"), C.c_size_t]
    lib.ref_write_component.restype = C.c_size_t
    lib.ref_intra_case.argtypes = [C.c_int, C.POINTER(abi.Geom), PL, PL, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    lib.ref_film_grain.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, PL, C.POINTER(C.c_ssize_t)] + [C.c_void_p] * 4 + [C.POINTER(C.c_int), C.c_void_p]
    lib.ref_picture_hash.argtypes = [C.c_int, C.c_int, PL, C.POINTER(C.c_ssize_t), C.c_int, C.c_int, np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS"), C.c_int]
    lib.ref_lmcs_build.argtypes = [C.c_int] * 3 + [C.POINTER(C.c_int), C.c_int, C.c_int, C.POINTER(abi.Lmcs), i16p]
    lib.ref_lmcs_fwd_block.argtypes = [C.c_int, V, C.c_ssize_t, C.c_int, C.c_int]
    lib.ref_lmcs_inv_block.argtypes = [C.c_int, V, C.c_ssize_t, C.c_int, C.c_int]
    lib.ref_lmcs_scale_block.argtypes = [V, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.ref_lmcs_vpdu_scale.argtypes = [C.POINTER(abi.Geom), PL, C.c_int, C.c_int]
    lib.ref_decompress_picture_out.argtypes = [C.POINTER(abi.Geom), C.POINTER(C.c_void_p), C.POINTER(abi.Picture), C.c_int, C.c_int, PL]
    lib.ref_decompress_picture_out.restype = C.c_double
    lib.ref_decompress_picture_mt.argtypes = [C.POINTER(abi.Geom), C.POINTER(C.c_void_p), C.POINTER(abi.Picture), C.c_int, C.c_int]
    lib.ref_decompress_picture_mt.restype = C.c_double
    declare_seam(lib)
    return lib


# ---- the DecLibRecon seam (oracle/ref_seam.h) ----
SEAM = dict(BDOF=1, DMVR=2, BCW=4, PROF=8, MMVD=16, GEO=32, CIIP=64, SMVD=128, AMVR=256, MTS=512, LFNST=1024, SBT=2048, MRL=4096, MIP=8192, CCLM=16384,
            JCCR=32768, TS=65536, BDPCM=1 << 17, SAO=1 << 18, ALF=1 << 19, LMCS=1 << 20, DEPQUANT=1 << 21, LOCAL_DUAL_TREE=1 << 22, VIRTUAL_BOUNDARIES=1 << 23, NO_LF_ACROSS_SLICES=1 << 24, WP=1 << 25, SCALING_LIST=1 << 26)
SEAM_INTER_TOOLS = sum(SEAM[k] for k in ("BDOF", "DMVR", "BCW", "PROF", "MMVD", "GEO", "SMVD", "AMVR"))
SEAM_RESI_TOOLS = sum(SEAM[k] for k in ("MTS", "SBT", "JCCR", "TS", "DEPQUANT"))
SEAM_INTRA_TOOLS = sum(SEAM[k] for k in ("LFNST", "MRL", "MIP", "CCLM", "BDPCM", "CIIP"))
SEAM_FILTERS = SEAM["SAO"] | SEAM["ALF"]


class SeamCfg(C.Structure):
    _fields_ = [("seed", C.c_uint32)] + [(n, C.c_int32) for n in ("sliceType", "tools", "qp", "intraPct", "skipPct", "mergePct", "affinePct", "biPct", "rootCbfPct",
                                                                    "cbfPct", "splitPct", "ispPct", "mvdSigmaQpel", "lmcsMinBin", "lmcsMaxBin")] + \
               [("lmcsDeltaCW", C.c_int32 * 16), ("lmcsChrOffset", C.c_int32), ("lmcsChromaAdj", C.c_int32), ("numSlices", C.c_int32)]


def seam_cfg(seed, slice_type=0, tools=None, qp=32, intra=15, skip=15, merge=50, affine=12, bi=60, root_cbf=45, cbf=35, split=75, isp=0, mvd_sigma=12, lmcs=None, virtual_boundaries=False, slices=1, lf_across_slices=True, wp=False, scaling_lists=False):
    c = SeamCfg()
    c.seed = seed; c.sliceType = slice_type
    c.tools = (SEAM_INTER_TOOLS | SEAM_RESI_TOOLS | SEAM_INTRA_TOOLS | SEAM_FILTERS) if tools is None else tools
    c.qp = qp; c.intraPct = intra; c.skipPct = skip; c.mergePct = merge; c.affinePct = affine; c.biPct = bi; c.rootCbfPct = root_cbf; c.cbfPct = cbf
    c.splitPct = split; c.ispPct = isp; c.mvdSigmaQpel = mvd_sigma
    if virtual_boundaries: c.tools |= SEAM["VIRTUAL_BOUNDARIES"]
    c.numSlices = slices
    if not lf_across_slices: c.tools |= SEAM["NO_LF_ACROSS_SLICES"]
    if wp: c.tools |= SEAM["WP"]
    if scaling_lists: c.tools |= SEAM["SCALING_LIST"]
    if lmcs is not None:                                      # the dict synth.gen_lmcs returns
        c.tools |= SEAM["LMCS"]; c.lmcsMinBin = lmcs["minBin"]; c.lmcsMaxBin = lmcs["maxBin"]; c.lmcsChrOffset = lmcs["chrOff"]; c.lmcsChromaAdj = int(lmcs["struct"].chromaAdj)
        for i in range(16): c.lmcsDeltaCW[i] = lmcs["delta"][i]
    return c


def declare_seam(lib):
    if not hasattr(lib, "ref_seam_create"):
        return
    PL = C.POINTER(C.POINTER(C.c_int16))
    lib.ref_seam_create.argtypes = [C.POINTER(abi.Geom), C.POINTER(SeamCfg), C.POINTER(C.c_void_p), C.POINTER(abi.Picture)]; lib.ref_seam_create.restype = C.c_void_p
    lib.ref_seam_destroy.argtypes = [C.c_void_p]; lib.ref_seam_destroy.restype = None
    lib.ref_seam_col_motion_bytes.argtypes = [C.c_void_p]; lib.ref_seam_col_motion_bytes.restype = C.c_size_t
    lib.ref_seam_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]; lib.ref_seam_stats.restype = None
    lib.ref_seam_run_stock.argtypes = [C.c_void_p, C.c_int, PL, C.c_void_p, C.c_size_t]; lib.ref_seam_run_stock.restype = C.c_double
    lib.ref_seam_create_chained.argtypes = [C.POINTER(abi.Geom), C.POINTER(SeamCfg), C.POINTER(C.c_void_p), C.POINTER(abi.Picture), C.c_void_p]; lib.ref_seam_create_chained.restype = C.c_void_p
    lib.ref_seam_pipelined_flat.argtypes = [C.c_int, C.POINTER(abi.Picture)]; lib.ref_seam_pipelined_flat.restype = C.c_int
    lib.ref_seam_read_out.argtypes = [C.c_void_p, PL, C.c_void_p, C.c_size_t]; lib.ref_seam_read_out.restype = None
    lib.ref_seam_run_pipelined.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int]; lib.ref_seam_run_pipelined.restype = C.c_double
    lib.ref_seam_run_b200.argtypes = [C.c_void_p, C.c_int, C.c_int, PL, C.c_void_p, C.c_size_t, C.POINTER(abi.Picture)]; lib.ref_seam_run_b200.restype = C.c_double


def seam_pipelined(ref, cases, threads, backend, depth, read=True, chain=False, flat=False):
    """Runs the pictures of `cases` (SeamCase objects, one fresh Picture each) through `depth` alternating recon instances (ref_seam_run_pipelined).
    chain: every picture takes the one before it as its first list-0 reference (ref_seam_create_chained).  flat (dry-run back end, as many pictures as instances):
    also returns the work lists the instances flattened.  Returns (seconds, [(planes, colMotion) per picture][, lists])"""
    hs = []
    for c in cases: hs.append(c.build(prev=hs[-1] if chain and hs else None))
    arr = (C.c_void_p * len(hs))(*hs)
    secs = ref.ref_seam_run_pipelined(arr, len(hs), threads, backend, depth)
    outs = []
    if read and secs >= 0 and backend != 2:
        for c, h in zip(cases, hs):
            out = c._out(); col = np.zeros(ref.ref_seam_col_motion_bytes(h), np.uint8)
            ref.ref_seam_read_out(h, abi.plane_ptrs(out), col.ctypes.data, len(col)); outs.append((out, col))
    lists = []
    if flat and secs >= 0:
        for k, c in enumerate(cases):
            st = abi.Picture(); assert ref.ref_seam_pipelined_flat(k, C.byref(st)) == 0
            lists.append(picture_from_struct(st, c.g, c.filt))
    for h in reversed(hs): ref.ref_seam_destroy(h)
    return (secs, outs, lists) if flat else (secs, outs)


class SeamCase:
    """One synthetic parsed picture: geometry, reference pictures, filter parameters and generator configuration.  build() makes a fresh
    reference-side Picture from them (every back end consumes the one it reconstructs)."""
    def __init__(self, ref, rng, W, H, bd=10, ctu=128, lmcs=False, deblock=True, **cfg_kw):
        self.ref, self.g, self.W, self.H, self.bd = ref, abi.make_geom(W, H, bd, ctu=ctu), W, H, bd
        seed = int(rng.integers(1, 1 << 30))
        self.refs = [synth.noise_planes(rng, W, H, bd) for _ in range(4)]
        # filter-stage parameters only: deblocking offsets, SAO, ALF (+ an LMCS model); the CU-level content comes from the seam generator
        self.filt = synth.gen_picture(rng, W, H, bd, ctu=ctu, dst_slot=4, inter=False, cu_kw=dict(min_dim=32, min_area=1024), tu_kw=dict(p_cbf=0.0), lmcs=lmcs, deblock=deblock)
        if deblock: self.filt["lfSlices"]["beta"] = rng.integers(-3, 4, size=(1, 3)); self.filt["lfSlices"]["tc"] = rng.integers(-3, 4, size=(1, 3))
        self.cfg = seam_cfg(seed, lmcs=self.filt.get("lmcs"), **cfg_kw)

    def variant(self, seed, slice_type=None):
        """Another picture with the same reference pictures and filter parameters: a different generator seed (and slice type)."""
        import copy
        v = copy.copy(self)
        v.cfg = SeamCfg.from_buffer_copy(self.cfg)
        v.cfg.seed = seed
        if slice_type is not None: v.cfg.sliceType = slice_type
        return v

    def build(self, prev=None):
        if prev is not None: h = self.ref.ref_seam_create_chained(C.byref(self.g), C.byref(self.cfg), ref_ptrs(self.refs), C.byref(self.filt["struct"]), prev)
        else: h = self.ref.ref_seam_create(C.byref(self.g), C.byref(self.cfg), ref_ptrs(self.refs), C.byref(self.filt["struct"]))
        assert h, "ref_seam_create failed"
        return h

    def stats(self):
        h = self.build(); st = (C.c_int32 * 16)(); self.ref.ref_seam_stats(h, st); self.ref.ref_seam_destroy(h)
        names = ["cus", "intra", "tus", "skip", "merge", "affine", "geo", "ciip", "mmvd", "resi", "sbt", "lfnst", "mts", "isp", "mip", "chromaTree"]
        return dict(zip(names, list(st)))

    def _out(self):
        return [np.zeros((self.H, self.W), np.int16), np.zeros((self.H // 2, self.W // 2), np.int16), np.zeros((self.H // 2, self.W // 2), np.int16)]

    def run_stock(self, threads=0):
        h = self.build(); out = self._out(); col = np.zeros(self.ref.ref_seam_col_motion_bytes(h), np.uint8)
        secs = self.ref.ref_seam_run_stock(h, threads, abi.plane_ptrs(out), col.ctypes.data, len(col))
        self.ref.ref_seam_destroy(h)
        assert secs >= 0, f"stock DecLibRecon failed ({secs})"
        return out, col, secs

    def run_b200(self, threads=0):
        h = self.build(); out = self._out(); col = np.zeros(self.ref.ref_seam_col_motion_bytes(h), np.uint8)
        secs = self.ref.ref_seam_run_b200(h, threads, 0, abi.plane_ptrs(out), col.ctypes.data, len(col), None)
        self.ref.ref_seam_destroy(h)
        return out, col, secs

    def flatten(self, threads=0):
        """Host stages of DecLibReconB200 only (no device): the work lists as a picture dict of copies, usable with helpers.oracle_decompress / the C ABI."""
        h = self.build(); flat = abi.Picture(); col = np.zeros(self.ref.ref_seam_col_motion_bytes(h), np.uint8)
        secs = self.ref.ref_seam_run_b200(h, threads, 1, None, col.ctypes.data, len(col), C.byref(flat))
        self.ref.ref_seam_destroy(h)
        if secs < 0: return None, secs
        pic = picture_from_struct(flat, self.g, self.filt); pic["colMotion"] = col            # colMotion: with zero DMVR deltas (no device in a dry run)
        return pic, secs


COL_MOTION_DTYPE = np.dtype([("mv", "<i4", (2, 2)), ("ref", "i1", (2,)), ("pad", "u1", (2,))])      # vvdec::ColocatedMotionInfo (MotionInfo.h:154), 20 bytes


def col_motion_diff(a, b, g=None):
    """Number of 8x8 entries whose collocated motion differs: reference indices, and MVs where the list is in use (the structs are copied with
    their padding, and the MV of an unused list is whatever the motion buffer held).  g: geometry — entries of the CTU-major map
    ([ctu][ctu/8][ctu/8]) that lie outside the picture are never written and are left out."""
    A, B = a.view(COL_MOTION_DTYPE), b.view(COL_MOTION_DTYPE)
    bad = (A["ref"] != B["ref"]).any(axis=1)
    if g is not None:
        n8 = g.ctuSize // 8; cw = (g.width + g.ctuSize - 1) // g.ctuSize
        idx = np.arange(len(A)); ctu, r = idx // (n8 * n8), idx % (n8 * n8)
        inside = ((ctu % cw) * g.ctuSize + (r % n8) * 8 < g.width) & ((ctu // cw) * g.ctuSize + (r // n8) * 8 < g.height)
    else:
        inside = np.ones(len(A), bool)
    bad &= inside
    for l in range(2):
        bad |= inside & (A["ref"][:, l] >= 0) & (A["mv"][:, l] != B["mv"][:, l]).any(axis=1)
    return int(bad.sum())


def _copy(ptr, n, dtype):
    if not n: return np.zeros(0, dtype)
    if not ptr: return np.zeros(n, dtype)                        # a table the picture does not use (e.g. no CC-ALF filters)
    return np.frombuffer((C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr), dtype=dtype).copy()


def picture_from_struct(st, g, filt):
    """Deep copy of a b200_picture (pointers into the recon object) into the dict layout of synth.gen_picture."""
    W4, H4 = (g.width + 3) // 4, (g.height + 3) // 4
    nctu = ((g.width + g.ctuSize - 1) // g.ctuSize) * ((g.height + g.ctuSize - 1) // g.ctuSize)
    d = dict(pus=_copy(st.pus, st.numPus, synth.PU_DTYPE), ndmvr=int(st.numDmvr) - 1, tus=_copy(st.tus, st.numTus, abi.TU_DTYPE), coefs=_copy(st.coefs, st.numCoefs, np.int16))
    if len(d["coefs"]) == 0: d["coefs"] = np.zeros(1, np.int16)
    if st.numScaling: d["scaling"] = _copy(st.scaling, st.numScaling, np.int32)
    p = abi.Picture(); p.dstSlot = st.dstSlot; p.flags = st.flags
    p.pus = d["pus"].ctypes.data; p.numPus = len(d["pus"]); p.numDmvr = st.numDmvr
    p.tus = d["tus"].ctypes.data; p.numTus = len(d["tus"]); p.coefs = d["coefs"].ctypes.data; p.numCoefs = st.numCoefs
    if st.numScaling: p.scaling = d["scaling"].ctypes.data; p.numScaling = st.numScaling
    if st.numIntraTus:
        d["intraTus"] = _copy(st.intraTus, st.numIntraTus, abi.INTRA_TU_DTYPE); p.intraTus = d["intraTus"].ctypes.data; p.numIntraTus = st.numIntraTus
    if st.flags & abi.PIC_DEBLOCK:
        d["lfV"] = _copy(st.lfV, W4 * H4, synth.LF_DTYPE); d["lfH"] = _copy(st.lfH, W4 * H4, synth.LF_DTYPE); d["lfSlices"] = _copy(st.lfSlices, st.numLfSlices, synth.LFSLICE_DTYPE)
        p.lfV = d["lfV"].ctypes.data; p.lfH = d["lfH"].ctypes.data; p.lfSlices = d["lfSlices"].ctypes.data; p.numLfSlices = st.numLfSlices
        if st.ctuSlice: d["ctuSlice"] = _copy(st.ctuSlice, nctu, np.uint8); p.ctuSlice = d["ctuSlice"].ctypes.data
        if st.lfSeq:                                             # luma-adaptive deblocking offsets of the SPS
            d["lfSeq"] = abi.LfSeq.from_buffer_copy(C.string_at(st.lfSeq, C.sizeof(abi.LfSeq))); p.lfSeq = C.addressof(d["lfSeq"])
    if st.flags & abi.PIC_SAO:
        d["sao"] = _copy(st.sao, nctu, synth.SAO_DTYPE); p.sao = d["sao"].ctypes.data
    if st.flags & abi.PIC_ALF:
        d["alf"] = dict(ctus=_copy(st.alf, nctu, synth.ALFCTU_DTYPE)); p.alf = d["alf"]["ctus"].ctypes.data
        T = C.cast(st.alfTabs, C.POINTER(abi.AlfTables)).contents
        d["alfArrays"] = dict(lumaCoeff=_copy(T.lumaCoeff, T.numLumaSets * 1300, np.int16), lumaClip=_copy(T.lumaClip, T.numLumaSets * 1300, np.int16),
                              chromaCoeff=_copy(T.chromaCoeff, max(1, T.numChromaAlts) * 7, np.int16), chromaClip=_copy(T.chromaClip, max(1, T.numChromaAlts) * 7, np.int16),
                              cc0=_copy(T.ccCoeff[0], max(1, T.numCc[0]) * 7, np.int16), cc1=_copy(T.ccCoeff[1], max(1, T.numCc[1]) * 7, np.int16))
        A = abi.AlfTables(); a = d["alfArrays"]
        A.lumaCoeff = a["lumaCoeff"].ctypes.data; A.lumaClip = a["lumaClip"].ctypes.data; A.numLumaSets = T.numLumaSets
        A.chromaCoeff = a["chromaCoeff"].ctypes.data; A.chromaClip = a["chromaClip"].ctypes.data; A.numChromaAlts = T.numChromaAlts
        A.ccCoeff[0] = a["cc0"].ctypes.data; A.ccCoeff[1] = a["cc1"].ctypes.data; A.numCc[0] = T.numCc[0]; A.numCc[1] = T.numCc[1]
        d["alfTabs"] = A; p.alfTabs = C.addressof(A)
    if st.numWp:
        d["wp"] = _copy(st.wp, st.numWp, synth.WP_DTYPE); p.wp = d["wp"].ctypes.data; p.numWp = st.numWp
    if st.flags & abi.PIC_LMCS:
        L = C.cast(st.lmcs, C.POINTER(abi.Lmcs)).contents
        vs = 64 if g.ctuSize == 128 else g.ctuSize
        nv = ((g.width + vs - 1) // vs) * ((g.height + vs - 1) // vs)
        L2 = abi.Lmcs(); C.memmove(C.byref(L2), C.byref(L), C.sizeof(abi.Lmcs))
        inv = _copy(L.invLUT, 1 << g.bitDepth, np.int16); vp = _copy(L.vpdus, nv, synth.LMCS_VPDU_DTYPE) if L.vpdus else np.zeros(nv, synth.LMCS_VPDU_DTYPE)
        L2.invLUT = inv.ctypes.data; L2.vpdus = vp.ctypes.data
        d["lmcs"] = dict(struct=L2, invLUT=inv, vpdus=vp); p.lmcs = C.addressof(L2)
    d["struct"] = p
    return d


def aligned(shape, dtype, fill=0, align=64):
    """numpy array whose data pointer is `align`-byte aligned (the reference's SIMD paths use aligned loads)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape))
    raw = np.zeros(n * dtype.itemsize + align, np.uint8)
    off = (-raw.ctypes.data) % align
    a = raw[off:off + n * dtype.itemsize].view(dtype).reshape(shape)
    a[...] = fill
    return a


def aligned_copy(src, align=64):
    a = aligned(src.shape, src.dtype, align=align)
    a[...] = src
    return a


def ref_ptrs(ref_pics):
    """ref_pics: list of [Y, Cb, Cr] int16 arrays per DPB slot -> (const int16_t* [slots*3])."""
    arr = (C.c_void_p * (3 * len(ref_pics)))()
    for s, pl in enumerate(ref_pics):
        for c in range(3):
            arr[s * 3 + c] = pl[c].ctypes.data
    return arr


def oracle_decompress(oracle, g, dpb, pic):
    """CPU chain of the whole back end on one synthetic picture: K2 -> K1 -> K3 -> K4 -> K5 with the pinned oracle.
    dpb: list of [Y,Cb,Cr] per slot (refs are read from it); returns the new picture planes and the DMVR deltas."""
    SC = pic["scaling"].ctypes.data if "scaling" in pic else None      # explicit scaling lists: the picture's dequantisation tables
    W, H = g.width, g.height
    cur = [np.zeros((H, W), np.int16), np.zeros((H // 2, W // 2), np.int16), np.zeros((H // 2, W // 2), np.int16)]
    dm = np.zeros((pic["ndmvr"] + 1, 2), np.int32)
    st = pic["struct"]
    if "given" in pic:                                          # pre-reconstructed (intra) samples: b200_picture::given
        cur = [p.copy() for p in pic["given"]]
    oracle.orc_mc_predict_wp(C.byref(g), abi.plane_ptrs(cur), ref_ptrs(dpb), pic["pus"].ctypes.data, len(pic["pus"]), dm.ctypes.data,
                             pic["wp"].ctypes.data if "wp" in pic else None)
    if st.flags & abi.PIC_LMCS and "intraTus" in pic:
        # LMCS with intra / CIIP blocks: everything before the inverse map lives in the mapped domain.  The chroma residual scale of a VPDU comes from its
        # reconstructed luma neighbourhood (intra blocks included), so: luma TUs -> luma intra blocks -> scales -> chroma TUs (scaled) -> chroma intra blocks
        L = C.byref(pic["lmcs"]["struct"]); chroma_adj = bool(pic["lmcs"]["struct"].chromaAdj)
        oracle.orc_lmcs_fwd_pus(C.byref(g), cur[0], pic["pus"].ctypes.data, len(pic["pus"]), L)
        resi = [np.zeros_like(p) for p in cur]
        it = pic["intraTus"]; it_y, it_c = np.ascontiguousarray(it[it["comp"] == 0]), np.ascontiguousarray(it[it["comp"] != 0])
        tus = pic["tus"]; n = len(tus)
        oracle.orc_k1_residual_sel(C.byref(g), abi.plane_ptrs(cur), abi.plane_ptrs(resi), tus.ctypes.data, n, pic["coefs"], SC, 1, None)
        oracle.orc_intra_reconstruct(C.byref(g), abi.plane_ptrs(cur), abi.plane_ptrs(resi), it_y.ctypes.data, len(it_y))
        vs = 64 if g.ctuSize == 128 else g.ctuSize
        scale = np.zeros(((W + vs - 1) // vs) * ((H + vs - 1) // vs), np.int32)
        if chroma_adj: oracle.orc_lmcs_vpdu_scales(C.byref(g), cur[0], L, scale.ctypes.data)
        oracle.orc_k1_residual_sel(C.byref(g), abi.plane_ptrs(cur), abi.plane_ptrs(resi), tus.ctypes.data, n, pic["coefs"], SC, 2, scale.ctypes.data if chroma_adj else None)
        oracle.orc_intra_reconstruct(C.byref(g), abi.plane_ptrs(cur), abi.plane_ptrs(resi), it_c.ctypes.data, len(it_c))
        oracle.orc_lmcs_inv_plane(C.byref(g), cur[0], L)
    elif st.flags & abi.PIC_LMCS:
        # DecCu.cpp:458-476 forward map of every inter CU's luma prediction; :483 finishLMCSAndReco; DecLibRecon.cpp:935 inverse map
        L = C.byref(pic["lmcs"]["struct"])
        oracle.orc_lmcs_fwd_pus(C.byref(g), cur[0], pic["pus"].ctypes.data, len(pic["pus"]), L)
        oracle.orc_k1_residual_lmcs(C.byref(g), abi.plane_ptrs(cur), pic["tus"].ctypes.data, len(pic["tus"]), pic["coefs"], SC, L)
        oracle.orc_lmcs_inv_plane(C.byref(g), cur[0], L)
    elif "intraTus" in pic:
        # intra CUs on the device: their TUs (TU_RESI) leave the residual in separate planes, K6 predicts + reconstructs them in decoding order
        tus = pic["tus"]; rs = (tus["flags"] & abi.TU_RESI) != 0
        t0, t1 = np.ascontiguousarray(tus[~rs]), np.ascontiguousarray(tus[rs])
        resi = [np.zeros_like(p) for p in cur]
        oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(cur), t0.ctypes.data, len(t0), pic["coefs"], SC, 0)
        oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(resi), t1.ctypes.data, len(t1), pic["coefs"], SC, 1)
        oracle.orc_intra_reconstruct(C.byref(g), abi.plane_ptrs(cur), abi.plane_ptrs(resi), pic["intraTus"].ctypes.data, len(pic["intraTus"]))
    else:
        oracle.orc_k1_residual(C.byref(g), abi.plane_ptrs(cur), pic["tus"].ctypes.data, len(pic["tus"]), pic["coefs"], SC, 0)
    if st.flags & abi.PIC_DEBLOCK:
        oracle.orc_lf_deblock(C.byref(g), abi.plane_ptrs(cur), pic["lfV"].ctypes.data, pic["lfH"].ctypes.data, pic["ctuSlice"].ctypes.data if "ctuSlice" in pic else None,
                              pic["lfSlices"].ctypes.data, C.byref(pic["lfSeq"]) if "lfSeq" in pic else None, 3)
    if st.flags & abi.PIC_SAO:
        nxt = [np.zeros_like(p) for p in cur]
        oracle.orc_sao_picture(C.byref(g), abi.plane_ptrs(cur), abi.plane_ptrs(nxt), pic["sao"].ctypes.data, None)
        cur = nxt
    if st.flags & abi.PIC_ALF:
        nxt = [np.zeros_like(p) for p in cur]
        oracle.orc_alf_picture(C.byref(g), abi.plane_ptrs(cur), abi.plane_ptrs(nxt), pic["alf"]["ctus"].ctypes.data, C.byref(pic["alfTabs"]))
        cur = nxt
    return cur, dm


def intra_picture_case(ref, rng, W, H, bd, ctu, simd, p_resi=0.5, colloc=0, **layout_kw):
    """A whole all-intra picture through the real IntraPrediction: every CU predicted from the reconstruction of the earlier ones, with the
    pred + residual step on some CUs.  Returns geometry, start planes, residual planes, records (from the reference's flattener) and the result."""
    g = abi.make_geom(W, H, bd, ctu=ctu)
    layout = synth.gen_intra_layout(rng, W, H, ctu, **layout_kw)
    planes = synth.noise_planes(rng, W, H, bd)
    resi = [rng.integers(-40, 41, size=p.shape).astype(np.int16) for p in planes]
    cus = np.zeros(len(layout), synth.REF_INTRA_CU_DTYPE)
    chroma = [0, 1, 18, 50, 2, 34, 66, 70, 70, 70, 23, 45, 61, 67, 67, 68, 69]      # 67..69: LM, MDLM_L, MDLM_T
    for i, (x, y, w, h) in enumerate(layout):
        cus[i]["x"], cus[i]["y"], cus[i]["w"], cus[i]["h"] = x, y, w, h
        cus[i]["dirL"], cus[i]["dirC"] = int(rng.integers(0, 67)), chroma[int(rng.integers(len(chroma)))]
        r = rng.random()
        if r < 0.15 and y % ctu: cus[i]["multiRefIdx"], cus[i]["dirL"] = int(rng.integers(1, 3)), int(rng.integers(1, 67))
        elif r < 0.25 and w <= 32 and h <= 32: cus[i]["bdpcm"] = int(rng.integers(1, 3))
        elif r < 0.45:                                               # matrix intra prediction
            n_modes = 16 if (w, h) == (4, 4) else 8 if (w == 4 or h == 4 or (w, h) == (8, 8)) else 6
            cus[i]["dirL"] = int(rng.integers(0, n_modes)); cus[i]["rsv"][2] = 1 | (int(rng.integers(0, 2)) << 1)
        cus[i]["rsv"][0] = w < 8 or (w // 2) * (h // 2) < 16
        cus[i]["rsv"][1] = rng.random() < p_resi
    out = [p.copy() for p in planes]
    recs = np.zeros(3 * len(layout), abi.INTRA_TU_DTYPE)
    n = ref.ref_intra_case(simd, C.byref(g), abi.plane_ptrs(out), abi.plane_ptrs(resi), cus.ctypes.data, len(layout), 1, recs.ctypes.data, len(recs), colloc)
    assert n > 0, n
    return g, planes, resi, recs[:n], out


# ---- K6 kernel choice: launch_intra reads B200_INTRA_KERNEL / B200_INTRA_ORDER on every launch
INTRA_KERNELS = ("auto", "v1", "v1_decode", "v2")
_INTRA_ENV = {"auto": {}, "v1": {"B200_INTRA_KERNEL": "v1"}, "v1_decode": {"B200_INTRA_KERNEL": "v1", "B200_INTRA_ORDER": "decode"}, "v2": {"B200_INTRA_KERNEL": "v2"}}


@contextlib.contextmanager
def intra_kernel(kernel):
    """While the block runs, K6 takes `kernel`: auto (chosen by list density), v1 (one CTA per block; wave-front tickets for dense lists, list order
    otherwise), v1_decode (v1, tickets in list order), v2 (CTU-resident; v1 where a plane stride is odd)."""
    keys = ("B200_INTRA_KERNEL", "B200_INTRA_ORDER")
    old = {k: os.environ.get(k) for k in keys}
    for k in keys: os.environ.pop(k, None)
    os.environ.update(_INTRA_ENV[kernel])
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None: os.environ.pop(k, None)
            else: os.environ[k] = v


def intra_run(b200, kernel, g, planes, recs, resi=None):
    """b200_intra_reconstruct (b200_intra_predict without residual planes) of `recs` on copies of `planes` under `kernel`; returns the planes."""
    import vvdec_b200
    got = [None if p is None else p.copy() for p in planes]
    with intra_kernel(kernel):
        if resi is None: vvdec_b200.check(b200.b200_intra_predict(C.byref(g), abi.plane_ptrs(got), recs.ctypes.data, len(recs)))
        else: vvdec_b200.check(b200.b200_intra_reconstruct(C.byref(g), abi.plane_ptrs(got), abi.plane_ptrs(resi), recs.ctypes.data, len(recs)))
    return got


def assert_planes_equal(got, want, what=""):
    """Bit-exact planes; a failure names the plane, the number of differing samples and the first four (y, x)."""
    for c, (a, b) in enumerate(zip(got, want)):
        if b is None: continue
        bad = np.argwhere(a != b)
        assert len(bad) == 0, (what, c, len(bad), bad[:4].tolist())


def intra_dense(g, n):
    """launch_intra's density rule: at least 48 records per 128x128 luma area picks the CTU-resident kernel under auto."""
    return n >= 48 * max(1, (g.width * g.height) >> 14)


def intra_ctu_counts(recs, ctu, W):
    """Records per CTU (chroma positions scaled to luma)."""
    sh = (recs["comp"] > 0).astype(np.int64)
    cw = (W + ctu - 1) // ctu
    return np.bincount(((recs["y"].astype(np.int64) << sh) // ctu) * cw + ((recs["x"].astype(np.int64) << sh) // ctu))


# K6 cases beyond the random all-intra pictures: geometry, formats, bit depths and capacity (name -> keyword arguments of intra_case)
INTRA_CASES = {
    "ctu32_256x128": dict(W=256, H=128, ctu=32, min_size=4, p_isp=0.3, seed=21),
    "ctu32_416x240": dict(W=416, H=240, ctu=32, min_size=4, p_isp=0.3, seed=22),
    "ctu64_200x136": dict(W=200, H=136, ctu=64, min_size=4, p_isp=0.3, seed=23),            # partial CTUs: 8 x 8 luma corner, 4-wide / 4-high chroma tiles
    "stride_420": dict(W=416, H=240, ctu=128, min_size=4, strides=(420, 210, 210), seed=24),   # even strides, not a multiple of 8 samples
    "stride_417": dict(W=416, H=240, ctu=128, min_size=4, strides=(417, 209, 209), seed=25),   # odd stride: v1 under every setting
    "yuv400_8bit": dict(W=256, H=128, ctu=128, min_size=4, bd=8, chroma=False, seed=26),
    "yuv400_12bit": dict(W=256, H=128, ctu=128, min_size=4, bd=12, chroma=False, seed=27),
    "8bit_832x480": dict(W=832, H=480, ctu=128, min_size=4, bd=8, p_mip=0.4, seed=28),
    "12bit_832x480": dict(W=832, H=480, ctu=128, min_size=4, bd=12, p_mip=0.4, seed=29),
    "ctu_1244_blocks": dict(W=256, H=128, ctu=128, min_size=8, p_split=1.0, p_isp=0.9, p_mip=0.0, p_mrl=0.0, p_bdpcm=0.0, p_lm=0.0, seed=7),
    "ctu_1024_blocks": dict(W=256, H=128, ctu=128, min_size=4, p_split=1.0, p_isp=0.9, p_mip=0.0, p_mrl=0.0, p_bdpcm=0.0, p_lm=0.0, seed=7),
    "sparse_1080p": dict(W=1920, H=1080, ctu=128, min_size=8, p_split=0.6, intra=0.15, p_ciip=0.1, seed=30),   # the intra / CIIP blocks of a B picture
}


def intra_case(W, H, ctu, seed, min_size=8, bd=10, chroma=True, strides=None, p_split=0.75, p_isp=0.0, p_mip=0.15, p_mrl=0.15, p_bdpcm=0.08, p_lm=0.25, intra=None, p_ciip=0.25):
    """A list of gen_intra_records on noise planes with residual planes: returns (geometry, planes, residual planes, records).  intra: fraction of
    intra CUs (the others are inter CUs, p_ciip of those with a CIIP block of weight 1..3); None: every CU is intra."""
    rng = np.random.default_rng(seed)
    g = abi.make_geom(W, H, bd, chroma_format=1 if chroma else 0, ctu=ctu, strides=strides)
    layout = synth.gen_intra_layout(rng, W, H, ctu, min_size=min_size, p_split=p_split)
    only, ciip = None, None
    if intra is not None:
        only = rng.random(len(layout)) < intra
        ciip = {i: int(rng.integers(1, 4)) for i, (x, y, w, h) in enumerate(layout) if not only[i] and w * h >= 64 and rng.random() < p_ciip}
        for i in ciip: only[i] = True
    recs = synth.gen_intra_records(rng, layout, W, H, p_resi=0.5, p_lm=p_lm if chroma else 0.0, p_isp=p_isp, p_mip=p_mip, p_mrl=p_mrl, p_bdpcm=p_bdpcm,
                                   colloc=seed & 1, only=only, ciip=ciip, ctu=ctu)
    if not chroma: recs = np.ascontiguousarray(recs[recs["comp"] == 0])
    planes = synth.noise_planes(rng, W, H, bd, chroma=chroma, strides=strides)
    resi = [rng.integers(-40, 41, size=p.shape).astype(np.int16) for p in planes]
    if not chroma: planes, resi = planes + [None, None], resi + [None, None]
    return g, planes, resi, recs


# ---- pictures in flight (tests/test_pipeline_*.py): short schedules of synthetic pictures with a DPB slot plan
# Kinds: I an intra picture (dense list: the CTU-resident K6 kernel), B a B picture with sparse intra blocks and CIIP blocks that carry a residual (the
# one-CTA-per-block kernel and the CIIP clear), L the same with LMCS and chroma scaling (K6 in two passes), P inter only (DMVR on many PUs), p a small
# inter picture (large CUs, few records).  Filters: D deblocking, S SAO, A ALF ('-': off).  Every picture references DPB slots 0..3.
PIPELINE_KINDS = {
    "I": dict(intra_frac=1.0),
    "B": dict(intra_frac=0.05, p_ciip=0.1, cu_kw=dict(min_size=16)),
    "L": dict(intra_frac=0.05, p_ciip=0.1, cu_kw=dict(min_size=16), lmcs=True, lmcs_chroma=True),
    "P": dict(pu_kw=dict(p_dmvr=0.6)),
    "p": dict(cu_kw=dict(min_dim=32, min_area=1024)),
}
PIPELINE_SLOTS = 6
PIPELINE_SCHEDULES = {   # name -> (W, H, seed, [(kind, dstSlot, filters)])
    "416x240": (416, 240, 1, [("I", 4, "DSA"), ("B", 5, "D-A"), ("B", 5, "DS-"), ("L", 0, "DSA"), ("P", 1, "---"), ("B", 2, "D--"), ("P", 4, "DSA"), ("L", 3, "-SA")]),
    "832x480": (832, 480, 2, [("P", 4, "DSA"), ("I", 5, "DSA"), ("B", 0, "D-A"), ("L", 0, "---"), ("P", 1, "DS-"), ("B", 4, "DSA")]),
    "1920x1080": (1920, 1080, 3, [("I", 4, "DSA"), ("B", 5, "DSA"), ("P", 0, "D--")]),
    # small inter pictures first, then larger lists into the same arenas; the first intra picture arrives while the inter pictures are in flight
    "grow_416x240": (416, 240, 4, [("p", 4, "---"), ("p", 5, "---"), ("B", 4, "DSA"), ("L", 5, "DSA"), ("I", 0, "DSA")]),
}


@functools.lru_cache(maxsize=None)
def pipeline_schedule(name):
    """The pictures of PIPELINE_SCHEDULES[name]: a dict with g, W, H, the initial DPB (PIPELINE_SLOTS noise pictures), kinds, dsts and pics
    (synth.gen_picture dicts, struct.dstSlot set)."""
    W, H, seed, steps = PIPELINE_SCHEDULES[name]
    rng = np.random.default_rng(seed)
    bd = 10
    dpb = [synth.noise_planes(rng, W, H, bd) for _ in range(PIPELINE_SLOTS)]
    pics = [synth.gen_picture(rng, W, H, bd, dst_slot=dst, deblock="D" in f, sao="S" in f, alf="A" in f, **PIPELINE_KINDS[k]) for k, dst, f in steps]
    return dict(name=name, g=abi.make_geom(W, H, bd), W=W, H=H, bd=bd, dpb=dpb, kinds=[k for k, _, _ in steps], dsts=[d for _, d, _ in steps], pics=pics)


def pipeline_refs(pic):
    """DPB slots the picture's PUs read."""
    r = pic["pus"]["refSlot"].ravel()
    return set(int(v) for v in r[r >= 0])


def arena_bytes(g, pic):
    """Size of the arena b200_pic_upload lays out for the picture (picture.cu: every array at a 256-byte boundary, 16 bytes of slack)."""
    a = lambda n: (n + 16 + 255) & ~255
    st = pic["struct"]
    n4 = ((g.width + 3) >> 2) * ((g.height + 3) >> 2)
    nctu = ((g.width + g.ctuSize - 1) // g.ctuSize) * ((g.height + g.ctuSize - 1) // g.ctuSize)
    db, sao, alf, lm = st.flags & abi.PIC_DEBLOCK, st.flags & abi.PIC_SAO, st.flags & abi.PIC_ALF, st.flags & abi.PIC_LMCS
    tab = 0
    if alf:
        t = pic["alf"]; tab = 2 * (2 * len(t["lumaCoeff"]) * 1300 + 2 * len(t["chromaCoeff"]) * 7 + len(t["cc"][0]) * 7 + len(t["cc"][1]) * 7)
    vs = 64 if g.ctuSize == 128 else g.ctuSize
    nv = ((g.width + vs - 1) // vs) * ((g.height + vs - 1) // vs)
    ni = int(st.numIntraTus)
    sizes = [st.numPus * 64, n4 * 4, 2 * 128 * 4, st.numTus * 4, st.numTus * 32, st.numCoefs * 2, st.numScaling * 4, n4 * 6 if db else 0, n4 * 6 if db else 0, nctu,
             nctu * 24 if sao else 0, nctu * 8 if alf else 0, tab, st.numDmvr * 8, st.numWp * 24, C.sizeof(abi.Lmcs) if lm else 0, (2 << g.bitDepth) if lm else 0,
             nv * 6 if lm else 0, nv * 4 if lm else 0, 0, ni * 16, (ni + 2) * 4 if ni else 0, (ni + 8 + 3 * nctu) * 4 if ni else 0]
    if ni:
        for k in range(3 if g.chromaFormat else 1):
            pw, ph, unit = (g.width, g.height, 4) if k == 0 else (g.width >> 1, g.height >> 1, 2)
            sizes.append(((pw + unit - 1) // unit) * ((ph + unit - 1) // unit) * 4)
    return sum(a(s) for s in sizes)


# ---- K2: one comparison for every MC test (tests/test_k2_*.py)
def mc_dst(g, fill=-1):
    """Destination planes of a geometry (its strides, None for absent chroma), filled with a sentinel so that a sample nobody wrote stands out."""
    out = [np.full((g.height, g.stride[0]), fill, np.int16)]
    for c in (1, 2):
        out.append(np.full((g.height >> 1, g.stride[c]), fill, np.int16) if g.chromaFormat else None)
    return out


def mc_oracle(oracle, case):
    """orc_mc_predict_wp on a sweep case (synth.mc_sweep): (planes, DMVR deltas)."""
    g, pus = case["g"], case["pus"]
    a = mc_dst(g); da = np.zeros((case["ndmvr"] + 1, 2), np.int32)
    ent = case["wp"][1] if case["wp"] else None
    oracle.orc_mc_predict_wp(C.byref(g), abi.plane_ptrs(a), ref_ptrs(case["refs"]), pus.ctypes.data, len(pus), da.ctypes.data, None if ent is None else ent.ctypes.data)
    return a, da


def mc_tile_path(case, i, tx, ty):
    """Which path tile (tx, ty) of PU i takes in k2_inter.cu: its list, and for each list of the PU whether the window of the initial MV is interior
    (word copies) or on the boundary (per-sample clamped copies), DMVR's fast or slow search window."""
    pu = case["pus"][i]; g = case["g"]
    lst = synth.mc_list_of(pu, tx, ty)
    if lst == 16: return "affine list (one thread per sample, clamped reads)"
    tw, th = min(16, int(pu["w"]) - 16 * tx), min(16, int(pu["h"]) - 16 * ty)
    even = all(s % 2 == 0 for s in case["strides"][:3 if case["chroma"] else 1])
    kinds = ("dmvr", "dmvr_chroma") if lst // 4 == 3 else ("luma", "chroma")
    parts = []
    for l in range(2):
        if pu["refSlot"][l] < 0: continue
        win = synth.mc_tile_windows(pu, l, tx, ty)
        for k in kinds[:2 if case["chroma"] else 1]:
            x0, x1, y0, y1 = synth.mc_window_margins(k, g.width, g.height, tw, th)
            x, y = win[k]
            inside = even and x0 <= x <= x1 and y0 <= y <= y1
            parts.append(f"L{l} {k} " + (("fast" if inside else "slow") + " search window" if k.startswith("dmvr") else "interior" if inside else "boundary"))
    return f"list {lst} (mode {lst // 4}, class {lst % 4}, tile {tw}x{th}); " + ", ".join(parts)


def mc_mismatch(case, a, b, da, db):
    """None when the planes and DMVR deltas agree; else a message naming the case, the first differing sample, its PU and its tile's path.  The whole
    rows are compared, stride padding included: both sides start from the same sentinel, so a store past a row's last sample shows."""
    g = case["g"]
    for c in range(3 if g.chromaFormat else 1):
        A, B = a[c], b[c]
        if not np.array_equal(A, B):
            d = np.argwhere(A != B); y, x = (int(v) for v in d[0]); sh = 1 if c else 0
            pus = case["pus"]
            hit = [i for i, p in enumerate(pus) if p["x"] >> sh <= x < (p["x"] + p["w"]) >> sh and p["y"] >> sh <= y < (p["y"] + p["h"]) >> sh]
            where = "no PU"
            if hit:
                i = hit[0]; p = pus[i]
                tx, ty = ((x << sh) - int(p["x"])) // 16, ((y << sh) - int(p["y"])) // 16
                where = f"PU {i} ({case['tags'][i]}) {p}; tile ({tx}, {ty}): {mc_tile_path(case, i, tx, ty)}"
            return f"{case['name']}: plane {c}: {len(d)} samples differ, first at (y={y}, x={x}): {A[y, x]} vs {B[y, x]}; {where}"
    if not np.array_equal(da, db):
        bad = np.argwhere((da != db).any(axis=1))[:, 0]
        return f"{case['name']}: DMVR deltas differ at entries {bad[:5].tolist()}: {da[bad[:5]].tolist()} vs {db[bad[:5]].tolist()}"
    return None


# ---- K3: one call shape for every deblocking test (tests/test_k3_*.py)
def lf_args(case, planes):
    """The leading arguments of orc_lf_deblock / b200_lf_deblock for a sweep case (synth.lf_sweep) on `planes`: geometry, planes, grids, ctuSlice, slices."""
    cs = case["ctuSlice"]
    return (C.byref(case["g"]), abi.plane_ptrs(planes), case["lfV"].ctypes.data, case["lfH"].ctypes.data, None if cs is None else cs.ctypes.data,
            case["slices"].ctypes.data)


def lf_oracle(oracle, case, dirs=3, planes=None):
    """orc_lf_deblock of a sweep case on copies of its planes (or of `planes`)."""
    out = [None if p is None else p.copy() for p in (planes or case["planes"])]
    oracle.orc_lf_deblock(*lf_args(case, out), C.addressof(case["seq"]), dirs)
    return out


def lf_mismatch(oracle, case, got, want, dirs=3):
    """None when the planes agree (stride padding included); else a message naming the case, the plane, the first differing sample and the decision
    lf_decisions gives each segment that may write it (with dirs 3, horizontal segments are classified on the oracle's vertical-only output)."""
    for c, (a, b) in enumerate(zip(got, want)):
        if b is None or np.array_equal(a, b): continue
        bad = np.argwhere(a != b); y, x = (int(v) for v in bad[0])
        seen = []
        for d in (0, 1):
            if not dirs & (1 << d): continue
            start = lf_oracle(oracle, case, 1) if d and dirs & 1 else case["planes"]
            recs = synth.lf_decisions(start, case["lfH" if d else "lfV"], d, case["g"], case["slices"], case["seq"], case["ctuSlice"])
            seen += [f"{'H' if d else 'V'} edge ({r['x']}, {r['y']}) {r['tag']}" for r in recs if r["comp"] == c and (y, x) in r["writes"]]
        return f"{case['name']}: plane {c}: {len(bad)} samples differ, first at (y={y}, x={x}): {a[y, x]} vs {b[y, x]}; written by: {seen or 'no classified segment'}"
    return None



# ---- CCLM records the rules refuse (rules.cuh intra_problem), each row breaking one clause of a valid LM record; by default the picture is 256 x 256
# with CTU 128, so a 64-wide or 64-high chroma block still fits one chroma CTU and only the CCLM clause refuses it (with a smaller CTU those rows are left out)
def cclm_refusal_rows(W=256, H=256, ctu=128):
    """(geometry, valid records, [(name, record, what b200_last_error() says)]): a valid 8x8 Cb / Cr LM block and the rows that break it."""
    g = abi.make_geom(W, H, 10, ctu=ctu)
    pw, ph = W // 2, H // 2
    ok = np.zeros(2, abi.INTRA_TU_DTYPE)
    for i, c in enumerate((1, 2)):
        ok[i]["x"], ok[i]["y"], ok[i]["log2w"], ok[i]["log2h"], ok[i]["comp"], ok[i]["mode"] = 16, 16, 3, 3, c, abi.INTRA_LM
        ok[i]["flags"] = abi.INTRA_AVAIL_TL | abi.INTRA_LM_ABOVE | abi.INTRA_LM_LEFT | abi.INTRA_ADD_RESI
        ok[i]["numAbove"], ok[i]["numLeft"], ok[i]["lmAbove"], ok[i]["lmLeft"] = 8, 8, 4, 4

    def row(name, what="bad CCLM block", **f):
        r = ok[0].copy()
        for k, v in f.items(): r[k] = v
        return name, r, what
    bare = dict(flags=0, numAbove=0, numLeft=0, lmAbove=0, lmLeft=0)
    rows = [row("lm_on_luma", comp=0, x=32, y=32, **bare)]
    if ctu == 128: rows += [row("chroma_64_wide", x=64, y=0, log2w=6, **bare), row("chroma_64_high", x=0, y=64, log2h=6, **bare)]
    rows += [
            row("lmAbove_over_w", lmAbove=9), row("lmLeft_over_h", lmLeft=9),
            row("lm_above_at_y0", y=0, flags=abi.INTRA_LM_ABOVE, numAbove=0, numLeft=0, lmLeft=0),
            row("lm_left_at_x0", x=0, flags=abi.INTRA_LM_LEFT, numAbove=0, numLeft=0, lmAbove=0),
            row("template_past_right", mode=abi.INTRA_MDLM_T, x=pw - 8, lmAbove=8, numAbove=4),
            row("template_past_bottom", mode=abi.INTRA_MDLM_L, y=ph - 8, lmLeft=8, numLeft=4),
            row("mode_73", "bad mode", mode=73)]
    return g, ok, rows
