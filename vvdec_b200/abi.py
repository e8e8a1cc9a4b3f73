"""ctypes mirror of include/vvdec_b200.h (the C-ABI structs). Keep in sync with the header."""
import ctypes as C
import numpy as np

TR_DCT2, TR_DCT8, TR_DST7 = 0, 1, 2
TU_TS, TU_BDPCM_H, TU_BDPCM_V, TU_SCALING, TU_RESI = 1, 2, 4, 8, 16


class Tu(C.Structure):
    _fields_ = [("x", C.c_uint16), ("y", C.c_uint16), ("log2w", C.c_uint8), ("log2h", C.c_uint8),
                ("comp", C.c_uint8), ("flags", C.c_uint8), ("maxX", C.c_uint8), ("maxY", C.c_uint8),
                ("trType", C.c_uint8), ("lfnst", C.c_uint8), ("ict", C.c_int8), ("rightShift", C.c_int8),
                ("inBits", C.c_uint8), ("scale", C.c_uint8), ("coefOff", C.c_uint32), ("slOff", C.c_uint32),
                ("rsv", C.c_uint32 * 2)]


TU_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("log2w", "u1"), ("log2h", "u1"), ("comp", "u1"), ("flags", "u1"),
                     ("maxX", "u1"), ("maxY", "u1"), ("trType", "u1"), ("lfnst", "u1"), ("ict", "i1"),
                     ("rightShift", "i1"), ("inBits", "u1"), ("scale", "u1"), ("coefOff", "<u4"), ("slOff", "<u4"),
                     ("rsv", "<u4", (2,))])
assert TU_DTYPE.itemsize == C.sizeof(Tu) == 32


class Geom(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("chromaFormat", C.c_int32), ("bitDepth", C.c_int32),
                ("ctuSize", C.c_int32), ("stride", C.c_int32 * 3)]


def make_geom(width, height, bit_depth=10, chroma_format=1, ctu=128, strides=None):
    g = Geom(width, height, chroma_format, bit_depth, ctu)
    cw = width >> 1 if chroma_format == 1 else 0
    s = strides or (width, cw, cw)
    g.stride[0], g.stride[1], g.stride[2] = s
    return g


def plane_ptrs(planes):
    """planes: list of 3 contiguous int16 numpy arrays (or None). Returns (int16* [3])."""
    arr = (C.POINTER(C.c_int16) * 3)()
    for i, p in enumerate(planes):
        if p is not None:
            assert p.dtype == np.int16 and p.flags["C_CONTIGUOUS"]
            arr[i] = p.ctypes.data_as(C.POINTER(C.c_int16))
    return arr


class LfSeq(C.Structure):
    _fields_ = [("ladfEnabled", C.c_int32), ("ladfNumIntervals", C.c_int32), ("ladfQpOffset", C.c_int32 * 5),
                ("ladfIntervalLowerBound", C.c_int32 * 5)]


class Vb(C.Structure):
    _fields_ = [("numVer", C.c_int32), ("numHor", C.c_int32), ("posX", C.c_int32 * 3), ("posY", C.c_int32 * 3)]


class AlfTables(C.Structure):
    _fields_ = [("lumaCoeff", C.c_void_p), ("lumaClip", C.c_void_p), ("numLumaSets", C.c_int32),
                ("chromaCoeff", C.c_void_p), ("chromaClip", C.c_void_p), ("numChromaAlts", C.c_int32),
                ("ccCoeff", C.c_void_p * 2), ("numCc", C.c_int32 * 2)]


def make_alf_tables(t):
    """t: dict from synth.gen_alf (arrays must stay alive while the struct is used)."""
    T = AlfTables()
    T.lumaCoeff = t["lumaCoeff"].ctypes.data; T.lumaClip = t["lumaClip"].ctypes.data; T.numLumaSets = t["lumaCoeff"].shape[0]
    T.chromaCoeff = t["chromaCoeff"].ctypes.data; T.chromaClip = t["chromaClip"].ctypes.data; T.numChromaAlts = t["chromaCoeff"].shape[0]
    for c in range(2):
        T.ccCoeff[c] = t["cc"][c].ctypes.data; T.numCc[c] = t["cc"][c].shape[0]
    return T


def const_plane_ptrs(planes):
    return plane_ptrs(planes)


PIC_DEBLOCK, PIC_SAO, PIC_ALF, PIC_LMCS, PIC_DERIVE_LF = 1, 2, 4, 8, 16

# B200_PIC_DERIVE_LF records (b200_lf_cu, b200_lf_tu)
LF_CU_INTRA, LF_CU_CIIP, LF_CU_AFFINE, LF_CU_SBTMVP, LF_CU_GEO, LF_CU_ISP, LF_CU_BDPCM_Y, LF_CU_BDPCM_C, LF_CU_AVAIL_LEFT, LF_CU_AVAIL_TOP, LF_CU_SEP_TREE = \
    1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024
LF_CU_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("w", "u1"), ("h", "u1"), ("chType", "u1"), ("treeType", "u1"), ("flags", "<u2"), ("qp", "i1"),
                        ("slice", "u1"), ("geoLists", "u1"), ("numTus", "u1"), ("rsv", "u1", (2,)), ("firstTu", "<u4"), ("firstPu", "<u4")])
LF_TU_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("w", "u1"), ("h", "u1"), ("cx", "<u2"), ("cy", "<u2"), ("cw", "u1"), ("ch", "u1"),
                        ("cbf", "u1"), ("jointCbCr", "u1"), ("chromaQp", "i1", (2,))])
assert LF_CU_DTYPE.itemsize == 24 and LF_TU_DTYPE.itemsize == 16
LF_PARAM_DTYPE = np.dtype([("qp", "i1", (3,)), ("bs", "u1"), ("sideMaxFiltLength", "u1"), ("flags", "u1")])


class Picture(C.Structure):
    _fields_ = [("dstSlot", C.c_int32), ("flags", C.c_int32), ("given", C.c_void_p * 3),
                ("pus", C.c_void_p), ("numPus", C.c_size_t), ("numDmvr", C.c_size_t),
                ("tus", C.c_void_p), ("numTus", C.c_size_t), ("coefs", C.c_void_p), ("numCoefs", C.c_size_t),
                ("scaling", C.c_void_p), ("numScaling", C.c_size_t),
                ("lfV", C.c_void_p), ("lfH", C.c_void_p), ("ctuSlice", C.c_void_p), ("lfSlices", C.c_void_p),
                ("numLfSlices", C.c_int32), ("lfSeq", C.c_void_p),
                ("sao", C.c_void_p), ("vb", C.c_void_p), ("alf", C.c_void_p), ("alfTabs", C.c_void_p), ("wp", C.c_void_p), ("numWp", C.c_int32), ("lmcs", C.c_void_p),
                ("intraTus", C.c_void_p), ("numIntraTus", C.c_size_t),
                ("lfCus", C.c_void_p), ("numLfCus", C.c_size_t), ("lfTus", C.c_void_p), ("numLfTus", C.c_size_t),
                ("lfCtuCus", C.c_void_p), ("lfSliceB", C.c_void_p)]


class LmcsVpdu(C.Structure):
    _fields_ = [("x", C.c_uint16), ("y", C.c_uint16), ("availLeft", C.c_uint8), ("availAbove", C.c_uint8)]


class IntraTu(C.Structure):
    """b200_intra_tu (see include/vvdec_b200.h)."""
    _fields_ = [("x", C.c_uint16), ("y", C.c_uint16), ("log2w", C.c_uint8), ("log2h", C.c_uint8), ("comp", C.c_uint8), ("mode", C.c_uint8),
                ("multiRefIdx", C.c_uint8), ("flags", C.c_uint8), ("numAbove", C.c_uint8), ("numLeft", C.c_uint8), ("mip", C.c_uint8), ("lmAbove", C.c_uint8), ("lmLeft", C.c_uint8), ("ciip", C.c_uint8)]


INTRA_TU_DTYPE = np.dtype([("x", "<u2"), ("y", "<u2"), ("log2w", "u1"), ("log2h", "u1"), ("comp", "u1"), ("mode", "u1"), ("multiRefIdx", "u1"), ("flags", "u1"),
                           ("numAbove", "u1"), ("numLeft", "u1"), ("mip", "u1"), ("lmAbove", "u1"), ("lmLeft", "u1"), ("ciip", "u1")])
INTRA_FILTER_REF, INTRA_AVAIL_TL, INTRA_ADD_RESI = 1, 2, 4
INTRA_BDPCM_HOR, INTRA_BDPCM_VER, INTRA_MIP, INTRA_LM, INTRA_MDLM_L, INTRA_MDLM_T = 67, 68, 69, 70, 71, 72
INTRA_LM_ABOVE, INTRA_LM_LEFT, INTRA_LM_COLLOCATED, INTRA_ISP = 8, 16, 32, 64
ALF_CLIP_TOP, ALF_CLIP_BOTTOM, ALF_CLIP_LEFT, ALF_CLIP_RIGHT, ALF_PAD_TL, ALF_PAD_BR, ALF_PAD_WIDE = 2, 4, 8, 16, 32, 64, 2


class FilmGrain(C.Structure):
    """b200_film_grain: FilmGrainImpl's tables + the frame's line seeds (see include/vvdec_b200.h)."""
    _fields_ = [("pattern", C.c_void_p), ("sLUT", C.c_void_p), ("pLUT", C.c_void_p), ("lineSeeds", C.c_void_p),
                ("scaleShift", C.c_uint8), ("compPresent", C.c_uint8 * 3)]


class Lmcs(C.Structure):
    """b200_lmcs: the tables Reshape::constructReshaper derives (see include/vvdec_b200.h)."""
    _fields_ = [("chromaAdj", C.c_int32), ("minBinIdx", C.c_int32), ("maxBinIdx", C.c_int32), ("orgCW", C.c_int32),
                ("reshapePivot", C.c_int16 * 17), ("inputPivot", C.c_int16 * 17), ("fwdScaleCoef", C.c_int16 * 16),
                ("chromaAdjHelpLUT", C.c_int32 * 16), ("invLUT", C.c_void_p), ("vpdus", C.c_void_p)]
