/* vvdec_b200.h — C ABI of the GPU-native (H100, sm_90a) VVC pixel-reconstruction back end.
 *
 * Boundary (SURVEY.md §8b): this library replaces the *pixel work* behind VVdeC's
 * DecLibRecon::decompressPicture (reference: source/Lib/DecoderLib/DecLibRecon.cpp:429) and the
 * scalar/SIMD function-pointer surface of CommonLib (TrQuant/Quant/TCoeffOps, InterpolationFilter,
 * InterPrediction, LoopFilter, SampleAdaptiveOffset, AdaptiveLoopFilter).  VVdeC's parser keeps
 * running on the CPU; a host-side flattener turns each parsed Picture into the SoA work lists
 * declared here (plain pointers + sizes, no C++/torch types).
 *
 * Two levels of entry points:
 *   (1) picture level  — b200_ctx_*, b200_pic_* : the DecLibRecon seam (create / decompressPicture /
 *       waitForPrevDecompressedPic), operating on a decoded-picture buffer resident in HBM;
 *   (2) kernel level   — b200_k1_*, b200_if_*, b200_lf_*, b200_sao_*, b200_alf_* : host-pointer
 *       batch wrappers with the argument meaning of the reference pointer they replace, used by the
 *       parity tests exactly like vvdec_unit_test compares `ref` against `opt`.
 *
 * Every function returns 0 on success, a negative B200_ERR_* otherwise; b200_last_error() gives text.
 * All sample planes are int16 ("Pel", reference TypeDef.h:188), 4:2:0 or 4:0:0, bit depth 8..12.
 */
#ifndef VVDEC_B200_H
#define VVDEC_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_API __attribute__((visibility("default")))

enum {
  B200_OK            =  0,
  B200_ERR_CUDA      = -1,   /* a CUDA runtime call failed (maps to vvdec Exception, SURVEY §5) */
  B200_ERR_PARAM     = -2,   /* invalid argument (maps to RecoverableException)                */
  B200_ERR_NO_DEVICE = -3,   /* no sm_90 device:  the product path refuses to run on the CPU   */
  B200_ERR_UNSUPPORTED = -4  /* maps to UnsupportedFeatureException                            */
};

B200_API const char* b200_last_error(void);
B200_API int         b200_device_count(void);
B200_API const char* b200_version(void);

/* ------------------------------------------------------------------------------------------------
 * K1  residual: dequant + LFNST + inverse DCT-2/DST-7/DCT-8 + transform skip + BDPCM + joint CbCr
 *   replaces  Quant::DeQuant* (Quant.h:143-147, Quant.cpp:122-179, :295), invResDPCM (Quant.cpp:239),
 *             TrQuant::m_invLfnstNxN + xInvLfnst (TrQuant.cpp:79,:201), TrQuant::xIT (:410),
 *             fastInvTrans[][] / TCoeffOps::fastInvCore / roundClip / cpyResiClip (TrQuant_EMT.cpp),
 *             xITransformSkip (:489), invTransformCbCr (:108).
 * One record per coded TU component (what reconstructResi, DecCu.cpp:536, iterates).
 * ---------------------------------------------------------------------------------------------- */
enum { B200_TR_DCT2 = 0, B200_TR_DCT8 = 1, B200_TR_DST7 = 2 };          /* == vvdec TransType */
enum {
  B200_TU_TS       = 1,   /* mtsIdx == MTS_SKIP                                   */
  B200_TU_BDPCM_H  = 2,   /* bdpcmMode == 1 (accumulate along x), implies TS      */
  B200_TU_BDPCM_V  = 4,   /* bdpcmMode == 2 (accumulate along y), implies TS      */
  B200_TU_SCALING  = 8,   /* explicit scaling list: per-position factor at slOff  */
  B200_TU_RESI     = 16   /* picture path: TU of an intra CU — the residual goes to the picture's residual planes and K6
                             (b200_picture::intraTus, B200_INTRA_ADD_RESI) reconstructs the block in decoding order */
};

typedef struct b200_tu {
  uint16_t x, y;          /* top-left in the component's plane, samples                                  */
  uint8_t  log2w, log2h;  /* 1..6                                                                        */
  uint8_t  comp;          /* 0 Y, 1 Cb, 2 Cr : plane that receives the (first) residual                  */
  uint8_t  flags;         /* B200_TU_*                                                                   */
  uint8_t  maxX, maxY;    /* tu.maxScanPosX/Y[comp] (Unit.h:291); BDPCM: w-1,h-1                         */
  uint8_t  trType;        /* hor | ver<<2, B200_TR_* — result of TrQuant::getTrTypes (TrQuant.cpp:330)   */
  uint8_t  lfnst;         /* 0 off, else lfnstIdx(1|2) | set<<2 (g_lfnstLut[mode], 0..3) | transpose<<4  */
  int8_t   ict;           /* TU::getICTMode in -3..3 (0: none): also derive the other chroma plane       */
  int8_t   rightShift;    /* Quant::dequant's rightShift (Quant.cpp:337); <=0 means left shift           */
  uint8_t  inBits;        /* targetInputBitDepth (Quant.cpp:347): level clip to +-2^(inBits-1)           */
  uint8_t  scale;         /* g_InvQuantScales[sqrt2][QP_rem] (Quant.cpp:341)                             */
  uint32_t coefOff;       /* first level of the packed (maxX+1)x(maxY+1) corner, int16 units, row-major  */
  uint32_t slOff;         /* B200_TU_SCALING: int32 units into the scaling arena, w*h factors row-major  */
  uint32_t rsv[2];
} b200_tu;                /* 32 bytes */

/* Picture geometry shared by all stages. Planes have no margin: kernels clamp coordinates, which is
 * what the reference's 144-sample border extension (Picture.cpp:400-558) emulates.  Every entry point that takes a geometry returns
 * B200_ERR_PARAM for one outside these ranges, a width or height that is not a multiple of 8, or a plane stride below its plane's
 * width (SAO and ALF also need every stride to be a multiple of 4, ALF a bit depth of at most 10). */
typedef struct b200_geom {
  int32_t width, height;       /* luma samples                       */
  int32_t chromaFormat;        /* 0 = 4:0:0, 1 = 4:2:0               */
  int32_t bitDepth;            /* 8..12                              */
  int32_t ctuSize;             /* 32/64/128                          */
  int32_t stride[3];           /* samples per row of each plane      */
} b200_geom;

/* Kernel-level K1: host planes in, host planes out (in place).
 *   mode 0: planes hold the prediction; result = clip(pred + residual, 0, 2^bd-1)   (DecCu.cpp:455-479 reco)
 *   mode 1: result = residual only (what invTransformNxN leaves in pResi), planes pre-filled are overwritten
 *           only inside coded TUs.
 * Returns B200_ERR_PARAM, before any device work and with the planes untouched, for an invalid geometry (b200_geom) and for any TU the
 * picture path's list validation refuses. */
B200_API int b200_k1_residual(const b200_geom* g, int16_t* const planes[3],
                              const b200_tu* tus, size_t numTus,
                              const int16_t* coefs, size_t numCoefs,
                              const int32_t* scaling, size_t numScaling,
                              int mode);

/* ------------------------------------------------------------------------------------------------
 * K3  deblocking: all vertical edges of the picture, then all horizontal edges, in place.
 *   replaces  LoopFilter::loopFilterCTU / xDeblockCtuArea (LoopFilter.cpp:375,:418), xEdgeFilterLuma (:1463),
 *             xEdgeFilterChroma (:1619), LoopFilter::xPelFilterLuma (LoopFilter.h:106; xPelFilterLumaCore :213),
 *             LoopFilter::xFilteringPandQ (LoopFilter.h:122; xFilteringPandQCore :129), xPelFilterChroma (:281),
 *             xUseStrongFiltering (:1410), xCalcDP/DQ (:1392), deriveLADFShift (:1363).
 *   stays CPU: calcFilterStrengthsCTU (:360) — it produces the grid below from the CU/TU tree (SURVEY a14'), unless the picture asks the device
 *             to derive the grids from CU / TU records (B200_PIC_DERIVE_LF, b200_lf_derive below).
 * The edge grids are the reference's LoopFilterParam arrays (TypeDef.h:694, DecLibRecon.cpp:515) re-laid as one
 * picture-wide raster per direction: entry (x4,y4) describes the edge on the LEFT (lfV) / TOP (lfH) of the 4x4
 * luma unit at (4*x4, 4*y4).  Chroma uses the same entries on its 8x8-sample grid (LoopFilter.cpp:462-488).
 * ---------------------------------------------------------------------------------------------- */
typedef struct b200_lf_param {      /* == vvdec::LoopFilterParam, 6 bytes */
  int8_t  qp[3];                    /* (QpP+QpQ+1)>>1 per component                                      */
  uint8_t bs;                       /* Bs: bits 0-1 Y, 2-3 Cb, 4-5 Cr                                    */
  uint8_t sideMaxFiltLength;        /* (P<<4)|Q luma max filter lengths (1,2,3,5,7); bit 7 ignored       */
  uint8_t flags;                    /* bit 5: chroma "large" edge (both sides >= 8 chroma samples)       */
} b200_lf_param;

typedef struct b200_lf_slice {      /* Slice deblocking syntax (Slice.h getDeblockingFilter*)            */
  int8_t  betaOffsetDiv2[3];        /* Y, Cb, Cr                                                         */
  int8_t  tcOffsetDiv2[3];
  uint8_t disable;                  /* slice_deblocking_filter_disabled_flag                             */
  uint8_t rsv;
} b200_lf_slice;

typedef struct b200_lf_seq {        /* SPS luma-adaptive deblocking (LADF), Slice.h:1807-1813            */
  int32_t ladfEnabled, ladfNumIntervals;
  int32_t ladfQpOffset[5];
  int32_t ladfIntervalLowerBound[5];
} b200_lf_seq;

/* Kernel-level K3 on host planes (in place). lfV/lfH: [H/4][W/4] rasters. ctuSlice: slice index of
 * every CTU in raster order (NULL: all slice 0). seq may be NULL (LADF off). dirs: bit0 = vertical edges, bit1 = horizontal.
 * K3 filters all edges of one direction at once, which is exact only on a legal grid.  Per side, a luma edge of length n
 * writes n samples and reads 3, 3, 4, 6, 8 for n = 1, 2, 3, 5, 7; on a horizontal edge at a CTU row the P side counts as 3,
 * and when one side is long (5, 7) the other counts as at least 3.  A grid is legal when no Bs field is 3, no edge with
 * Bs != 0 lies on the picture's first column (lfV) / row (lfH), an edge with luma Bs != 0 has lengths 1, 2, 3, 5 or 7 and
 * reads nothing outside the picture, and any two luma edges e1 < e2 of one line (row of lfV, column of lfH) have
 * e2 - e1 >= writesQ(e1) + readsP(e2) and e2 - e1 >= readsQ(e1) + writesP(e2).  Edges of slices with deblocking disabled
 * count too.  Returns B200_ERR_PARAM, with the host planes untouched and the reason in b200_last_error(), for an illegal
 * grid, an invalid geometry (b200_geom), dirs & ~3, a ctuSlice entry >= numSlices, numSlices outside 1..64, or LADF with a
 * number of intervals outside 2..5.
 * The picture path (b200_picture::lfV / lfH) requires legal grids and does not check them; the grids the reference's
 * calcFilterStrengths derives, as the glue flattens them, are legal. */
B200_API int b200_lf_deblock(const b200_geom* g, int16_t* const planes[3], const b200_lf_param* lfV, const b200_lf_param* lfH,
                             const uint8_t* ctuSlice, const b200_lf_slice* slices, int numSlices, const b200_lf_seq* seq, int dirs);

/* Edge grids derived on the device (B200_PIC_DERIVE_LF): the picture carries its coding units and transform units instead of lfV / lfH, and
 * b200_pic_run derives both grids before K3 — LoopFilter::calcFilterStrengthsCTU (LoopFilter.cpp:360) with calcFilterStrengths (:495),
 * xSetMaxFilterLengthPQFromTransformSizes (:780), xSetMaxFilterLengthPQForCodingSubBlocks (:707), xSetEdgeFilterInsidePu (:1032) and
 * xGetBoundaryStrengthSingle (:1094), from a 4x4 motion field built out of the picture's b200_pu records (what MIDER stores, before the DMVR
 * deltas).  The grids are byte-identical to what the glue's flattenLfCtu copies out of the reference's per-CTU arrays.  IBC and virtual
 * boundaries are not part of it (the glue refuses both).
 * One b200_lf_cu per coding unit, in the order cs.traverseCUs walks each CTU, CTUs in raster order (b200_picture::lfCtuCus holds where each CTU's
 * CUs start); one b200_lf_tu per transform unit of a CU, coefficients or not, in the CU's TU order. */
enum {
  B200_LF_CU_INTRA = 1,       /* predMode MODE_INTRA (else MODE_INTER)                                                */
  B200_LF_CU_CIIP = 2, B200_LF_CU_AFFINE = 4, B200_LF_CU_SBTMVP = 8 /* merge type MRG_TYPE_SUBPU_ATMVP */, B200_LF_CU_GEO = 16,
  B200_LF_CU_ISP = 32,        /* ispMode() != 0                                                                        */
  B200_LF_CU_BDPCM_Y = 64, B200_LF_CU_BDPCM_C = 128,   /* bdpcmMode() / bdpcmModeChroma() != 0                          */
  B200_LF_CU_AVAIL_LEFT = 256, B200_LF_CU_AVAIL_TOP = 512,   /* xGetLoopfilterParam (:1063): leftEdge / topEdge            */
  B200_LF_CU_SEP_TREE = 1024  /* CU::isSepTree: the CU covers one channel type only                                    */
};
typedef struct b200_lf_cu {
  uint16_t x, y;              /* cu.blocks[chType]: position and size in samples of its channel type                  */
  uint8_t  w, h;
  uint8_t  chType;            /* 0 luma (with chroma unless B200_LF_CU_SEP_TREE), 1 chroma                             */
  uint8_t  treeType;          /* cu.treeType(): 0 TREE_D, 1 TREE_L, 2 TREE_C                                           */
  uint16_t flags;             /* B200_LF_CU_*                                                                          */
  int8_t   qp;                /* cu.qp                                                                                 */
  uint8_t  slice;             /* index into b200_picture::lfSlices / lfSliceB                                          */
  uint8_t  geoLists;          /* GEO: bit p = partition p predicts from list 1 (interDirrefIdxGeo0 / 1)                */
  uint8_t  numTus;            /* transform units of the CU: lfTus[firstTu .. firstTu + numTus - 1]                    */
  uint8_t  rsv[2];
  uint32_t firstTu;
  uint32_t firstPu;           /* inter CUs: its first b200_pu record (SbTMVP runs follow it); intra CUs: unused      */
} b200_lf_cu;                 /* 24 bytes */
typedef struct b200_lf_tu {
  uint16_t x, y; uint8_t w, h;        /* tu.blocks[Y] as the reference holds it (w = h = 0: no luma block)          */
  uint16_t cx, cy; uint8_t cw, ch;    /* tu.blocks[Cb] in chroma samples (cw = ch = 0: no chroma block)             */
  uint8_t  cbf;                       /* tu.cbf: bit c = coded block flag of component c                             */
  uint8_t  jointCbCr;
  int8_t   chromaQp[2];               /* tu.chromaQp (LoopFilter.cpp:1127-1128)                                      */
} b200_lf_tu;                         /* 16 bytes */
/* Kernel-level edge derivation: the lfV / lfH rasters ([H/4][W/4], host memory) of the records, derived on the device as b200_pic_run does for
 * B200_PIC_DERIVE_LF.  ctuCus: [number of CTUs + 1] as b200_picture::lfCtuCus; pus: the picture's b200_pu records (the motion field); slices / sliceB:
 * numSlices entries as b200_picture::lfSlices / lfSliceB.  Returns B200_ERR_PARAM, before any device work and with lfV / lfH untouched, for an invalid
 * geometry (b200_geom), numSlices outside 1..64, CTU ranges that do not run from 0 to numCus without going back, and a record the picture path refuses
 * too: a CU whose block (in its channel type) or one of whose TU blocks lies outside its plane or outside the CTU whose range lists the CU, an undefined
 * channel, tree type or flag, a slice index >= numSlices, no TU or TU records past numTus.  Records that pass but do not tile the picture the way a
 * coding tree does give undefined grids. */
struct b200_pu;
B200_API int b200_lf_derive(const b200_geom* g, const b200_lf_cu* cus, size_t numCus, const b200_lf_tu* tus, size_t numTus, const uint32_t* ctuCus,
                            const struct b200_pu* pus, size_t numPus, const b200_lf_slice* slices, const uint8_t* sliceB, int numSlices,
                            b200_lf_param* lfV, b200_lf_param* lfH);

/* ------------------------------------------------------------------------------------------------
 * K4  SAO: src (deblocked picture) -> dst, per CTU and component edge offset (4 directions) or band offset.
 *   replaces  SampleAdaptiveOffset::offsetBlock (SampleAdaptiveOffset.h:120; offsetBlock_core .cpp:64-349),
 *             SAOProcessCTU (:522), offsetCTU (:661), isProcessDisabled (:817).
 *   stays CPU: reconstructBlkSAOParam / merge resolution (:624) and deriveLoopFilterBoundaryAvailibility (:741) —
 *             the flattener stores their results in the per-CTU record below.
 * ---------------------------------------------------------------------------------------------- */
enum { B200_SAO_EO_0 = 0, B200_SAO_EO_90 = 1, B200_SAO_EO_135 = 2, B200_SAO_EO_45 = 3, B200_SAO_BO = 4, B200_SAO_OFF = 255 };
enum { B200_AVAIL_L = 1, B200_AVAIL_R = 2, B200_AVAIL_A = 4, B200_AVAIL_B = 8,
       B200_AVAIL_AL = 16, B200_AVAIL_AR = 32, B200_AVAIL_BL = 64, B200_AVAIL_BR = 128 };

typedef struct b200_sao_ctu {
  uint8_t type[3];        /* B200_SAO_* per component (typeIdc after merge resolution; OFF when modeIdc == SAO_MODE_OFF) */
  uint8_t band[3];        /* BO: typeAuxInfo = first band                                                               */
  int8_t  offset[3][5];   /* EO: offset[edgeType+2] (class order, PLAIN = 0); BO: offsets of bands band..band+3 in [0..3] */
  uint8_t avail;          /* B200_AVAIL_* of the 8 neighbouring CTUs (slice / tile / picture limits already applied)     */
  uint8_t rsv[2];
} b200_sao_ctu;           /* 24 bytes */

typedef struct b200_vb {  /* ph virtual boundaries (PicHeader), luma sample positions; used by SAO            */
  int32_t numVer, numHor;
  int32_t posX[3], posY[3];
} b200_vb;

/* Kernel-level K4: src planes -> dst planes (both host; dst must be a different buffer). vb may be NULL.  Only the plane width of each dst row is
 * written: the stride padding keeps what the caller put there.  Returns B200_ERR_PARAM, before any device work and with dst untouched, for a
 * chromaFormat other than 0 (4:0:0) or 1 (4:2:0), a CTU size other than 32 / 64 / 128, a bit depth outside 8..12, a width or height that is not a
 * multiple of 8, a plane stride below its plane's width or not a multiple of 4 (Cr included), a type other than 0..4 or B200_SAO_OFF, a BO band above
 * 31, more than 3 vertical or horizontal virtual boundaries, or a virtual boundary that is not a multiple of 8 strictly inside the picture.
 * The picture path (B200_PIC_SAO) refuses the same records in b200_pic_run, and the same geometry and virtual boundaries in b200_pic_upload;
 * VVC's virtual boundaries (at most 3 per direction, on the 8-sample grid) always meet these rules. */
B200_API int b200_sao_picture(const b200_geom* g, const int16_t* const src[3], int16_t* const dst[3],
                              const b200_sao_ctu* ctus, const b200_vb* vb);

/* ------------------------------------------------------------------------------------------------
 * K5  ALF + CC-ALF: src (SAO output) -> dst.
 *   replaces  AdaptiveLoopFilter::processCTU / filterCTU (AdaptiveLoopFilter.cpp:466,:664, the !isCrssByVBs path),
 *             m_deriveClassificationBlk (.h:128; .cpp:969), m_filter7x7Blk / m_filter5x5Blk (filterBlk<> :1175),
 *             m_filterCcAlf / m_filterCcAlfBoth (:1348,:1447), prepareCTU border extension (:453, here: clamping).
 *   stays CPU: reconstructCoeff(APSs) (:855,:888): the tables below are the *Final arrays it produces.
 *   not yet:   slices/tiles/subpictures with loop filtering disabled across them and explicit virtual
 *             boundaries (the isCrssByVBs path, :745-852) -> B200_ERR_UNSUPPORTED at the flattener.
 * ---------------------------------------------------------------------------------------------- */
/* CTUs whose neighbours ALF may not read (in-loop filtering disabled across slices / tiles: AdaptiveLoopFilter::isClipOrCrossedByVirtualBoundaries :118 and the
 * isCrssByVBs path of filterCTU :763-848): bits of b200_alf_ctu::enable[0].  CLIP_x: samples beyond that side of the CTU are replicas of its edge samples.
 * PAD_TL / PAD_BR (raster-scan slices: the CTU above-left / below-right belongs to another slice while both sides are readable): the corner region takes, row by
 * row, the sample of the CTU's first / last column (padBorderPel, Buffer.h:608).  enable[1], enable[2] bit 1 (B200_ALF_PAD_WIDE): the component is padded by 4 instead
 * of 2 chroma samples — what the reference does for a chroma component whose slice has CC-ALF off (AreaBuf::padBorderPel called with the luma margin, :794-803):
 * the region reaches 2 samples into the CTU and takes the sample 2 columns inside. */
enum { B200_ALF_CLIP_TOP = 2, B200_ALF_CLIP_BOTTOM = 4, B200_ALF_CLIP_LEFT = 8, B200_ALF_CLIP_RIGHT = 16, B200_ALF_PAD_TL = 32, B200_ALF_PAD_BR = 64, B200_ALF_PAD_WIDE = 2 };
typedef struct b200_alf_ctu {
  uint8_t enable[3];      /* alfCtuEnableFlag per component (bit 0); enable[0] bits 1..6: B200_ALF_CLIP_* / PAD_*, enable[1..2] bit 1: B200_ALF_PAD_WIDE */
  uint8_t lumaSet;        /* index into lumaCoeff/lumaClip: 0..15 fixed sets, 16.. the slice's APS sets        */
  uint8_t chromaAlt[2];   /* index into chromaCoeff/chromaClip (APS alternative, resolved per slice)           */
  uint8_t ccIdx[2];       /* 0: CC-ALF off for Cb/Cr, else 1 + index into ccCoeff[comp]                         */
} b200_alf_ctu;           /* 8 bytes */

typedef struct b200_alf_tables {
  const int16_t* lumaCoeff;    /* [numLumaSets][4 transposes][25 classes][13]  (lumaCoeffFinal / m_fixedFilterSetCoeffDec) */
  const int16_t* lumaClip;     /* same shape, clipping VALUES (lumaClippFinal / m_clipDefault)                              */
  int32_t        numLumaSets;
  const int16_t* chromaCoeff;  /* [numChromaAlts][7]                                                                        */
  const int16_t* chromaClip;   /* [numChromaAlts][7]                                                                        */
  int32_t        numChromaAlts;
  const int16_t* ccCoeff[2];   /* [numCc[c]][7]  (CcAlfFilterParam::ccAlfCoeff)                                             */
  int32_t        numCc[2];
} b200_alf_tables;

/* Kernel-level K5: src planes -> dst planes (both host).  Only the plane width of each dst row is written.  Returns B200_ERR_PARAM, before any device
 * work and with dst untouched, for the geometry b200_sao_picture refuses, a bit depth above 10 (ALF is defined for 8, 9 and 10 bit), numLumaSets
 * outside 16..24, a negative numChromaAlts or numCc (tables may hold several slices' APS filters), and for a CTU record with an enable bit outside the defined ones, lumaSet >=
 * numLumaSets (luma on), chromaAlt >= numChromaAlts (that chroma component on), ccIdx > numCc, PAD_TL together with CLIP_TOP or CLIP_LEFT or on the
 * picture's first CTU row or column, PAD_BR together with CLIP_BOTTOM or CLIP_RIGHT or on the last CTU row or column, or PAD_WIDE on a component
 * whose ccIdx is not 0.  The picture path (B200_PIC_ALF) refuses the same records in b200_pic_run, and the same geometry and table counts in
 * b200_pic_upload, except that its tables hold every slice's APS sets: numLumaSets may reach 255, the most a CTU record can address.  VVC's
 * tables (16 fixed luma sets and at most 8 APS sets per slice) always meet these rules. */
B200_API int b200_alf_picture(const b200_geom* g, const int16_t* const src[3], int16_t* const dst[3],
                              const b200_alf_ctu* ctus, const b200_alf_tables* tabs);

/* ------------------------------------------------------------------------------------------------
 * K2  inter prediction (motion compensation) into the current picture's planes.
 *   replaces  InterPrediction::motionCompensation (InterPrediction.cpp:1372) and below: xPredInterBi :686, xPredInterUni :623,
 *             xPredInterBlk :750, xSubPuBio :551 + applyBiOptFlow :1290 (BioGradFilter / BiOptFlow / PaddBIO pointers,
 *             InterPrediction.h:77-80,146), xProcessDMVR :1847 (xinitMC, xBIPMVRefine, xDMVRSubPixelErrorSurface, xPrefetchPad,
 *             xFinalPaddedMCForDMVR; RdCost SAD :107-221), xPredAffineBlk :934 (+ applyPROF / profGradFilter), xWeightedAverage
 *             :1346 (addAvg Buffer.cpp:441, addWeightedAvg :372), clipMvInPic (Mv.cpp:64), and the InterpolationFilter pointer
 *             table (InterpolationFilter.h:113-120; .cpp:424-962).
 *   stays CPU: merge/AMVP/affine/TMVP motion derivation (MIDER) and the mode decisions of motionCompensation :1411-1440
 *             (bioApplied, checkDMVRCondition UnitTools.cpp:1277, xCheckIdenticalMotion :404) — the flattener stores them as flags.
 *   also here: explicit weighted prediction (b200_wp), GEO blending (B200_PU_GEO); CIIP CUs take their inter half from here and the intra half from K6.
 *   not yet:   IBC, RPR-scaled references, wrap-around, sub-pictures.
 * One record per CU (ATMVP: per merged sub-PU run, InterPrediction.cpp:438). Reference pictures live in DPB slots.
 * ---------------------------------------------------------------------------------------------- */
enum {
  B200_PU_BDOF    = 1,    /* bioApplied (motionCompensation :1411-1428)                                          */
  B200_PU_DMVR    = 2,    /* dmvrApplied; refined MV deltas are written to dmvrMv[dmvrOff + subblock]             */
  B200_PU_ALTHPEL = 4,    /* cu.imv() == IMV_HPEL: alternative half-sample luma filter                            */
  B200_PU_AFFINE  = 8,    /* cu.affineFlag(): mv = CPMV0, cpmv = CPMV1/2; sub-block MVs as PU::setAllAffineMv     */
  B200_PU_AFFINE6 = 16,   /* 6-parameter model (else 4-parameter)                                                 */
  B200_PU_PROF0   = 32,   /* PROF enabled for list 0 / 1 (sps PROF && !ph dis_prof; the kernel applies the CPMV-equality and */
  B200_PU_PROF1   = 64,   /* spread-over-limit exclusions of xPredAffineBlk :1036-1040 itself)                     */
  B200_PU_GEO     = 128   /* cu.geoFlag(): geometric partitioning (motionCompensationGeo :1461, xWeightedGeoBlk
                             InterpolationFilter.cpp:1217).  refSlot[0]/mv[0] = partition 0 (interDirrefIdxGeo0, cu.mv[0][1]),
                             refSlot[1]/mv[1] = partition 1 (interDirrefIdxGeo1, cu.mv[1][1]) — both set, whatever lists they
                             come from; bcwW1 carries cu.geoSplitDir (0..63); w, h in 8..64                            */
};

typedef struct b200_pu {
  uint16_t x, y;            /* luma position                                                                       */
  uint8_t  w, h;            /* luma size, 4..128                                                                   */
  uint8_t  flags;           /* B200_PU_*                                                                           */
  int8_t   bcwW1;           /* weight of list 1 out of 8 (g_BcwWeights[g_BcwInternBcw[BcwIdx]]); 4 = plain average */
  int8_t   refSlot[2];      /* DPB slot of the reference picture per list; -1: list unused                         */
  uint8_t  interDir;        /* cu.interDir() (1 L0, 2 L1, 3 bi) — used by the affine spread check                  */
  uint8_t  wpIdx;           /* explicit weighted prediction: 1-based index into the picture's b200_wp table, 0 = none */
  uint32_t dmvrOff;         /* cu.mvdL0SubPuOff                                                                    */
  int32_t  mv[2][2];        /* [list][hor,ver] in 1/16 sample, as in cu.mv[list][0] (NOT clipped: kernels apply clipMvInPic) */
  int32_t  cpmv[2][2][2];   /* [list][1|2][hor,ver]: cu.mv[list][1], cu.mv[list][2] (affine only)                  */
} b200_pu;                  /* 64 bytes */

/* Explicit weighted prediction (reference CommonLib/WeightPrediction.cpp): one entry per (refIdx0, refIdx1) combination in use = what
 * WeightPrediction::getWpScaling (:67-147) returns for it.  Applies to translational and affine PUs without BDOF / DMVR / BCW
 * (InterPrediction.cpp:733-741: B slices with pps_weighted_bipred and BcwIdx == default, P slices with pps_weighted_pred).
 *   bi  (addWeightBi  :164): clip((w0*(P0+8192) + w1*(P1+8192) + (1 << s >> 1) + offset * (1 << (s-1))) >> s),  s = shift + max(2, 14-bd)
 *   uni (addWeightUni :238): clip(((w0*(P+8192) + (s ? 1 << (s-1) : 0)) >> s) + offset) */
typedef struct b200_wp {
  int16_t w0[3], w1[3];     /* per component; uni-prediction: w0 is the weight of the list in use                         */
  int16_t offset[3];        /* bi: o0 + o1, uni: o — iOffset << (bitDepth - 8)                                          */
  uint8_t shift[3];         /* bi: log2WeightDenom + 1, uni: log2WeightDenom                                            */
  uint8_t rsv[3];
} b200_wp;                  /* 24 bytes */

/* Kernel-level K2 on host planes: refs[slot*3 + comp] are the reference pictures (same geometry as g), dst the current
 * picture (only PU areas are written).  dmvrMv: int32 [n][2] (hor,ver deltas, Mv layout of m_dmvrMvCache), may be NULL. */
B200_API int b200_mc_predict(const b200_geom* g, int16_t* const dst[3], const int16_t* const* refs, int numSlots,
                             const b200_pu* pus, size_t numPus, int32_t* dmvrMv, size_t numDmvr);
/* the same with an explicit-weighted-prediction table (wp may be NULL when no PU has wpIdx != 0).
 * Both return B200_ERR_PARAM, before any device work and with dst and dmvrMv untouched, for an invalid geometry (b200_geom), and for any PU the
 * picture path's list validation refuses: reference slots outside [0, numSlots) or none, a side that is not a
 * multiple of 4 in 4..128 or leaves a 12-sample tile (12, 28, 44, ...), a block off the 4x4 grid or outside the picture, DMVR entries past numDmvr, DMVR on a uni-predicted, affine or
 * smaller than 8x8 / 128-sample PU, BDOF on such a small bi-predicted PU, DMVR above 10 bit, GEO that is uni-predicted, outside 8..64 per side,
 * combined with DMVR / BDOF / affine / weights or with a split direction above 63, and weights (wpIdx) past numWp or combined with DMVR, BDOF or BCW. */
B200_API int b200_mc_predict_wp(const b200_geom* g, int16_t* const dst[3], const int16_t* const* refs, int numSlots,
                                const b200_pu* pus, size_t numPus, int32_t* dmvrMv, size_t numDmvr, const b200_wp* wp, int numWp);

/* ------------------------------------------------------------------------------------------------
 * K6  intra prediction of one transform block (SURVEY 8f-1): regular modes, matrix intra prediction, cross-component linear model.
 *   replaces  IntraPrediction::initIntraPatternChType (IntraPrediction.cpp:947) = xFillReferenceSamples :1072 (the sample copies /
 *             substitution, not the availability analysis) + xFilterReferenceSamples :1251, and IntraPrediction::predIntraAng :474 =
 *             xPredIntraPlanarCore :154, xPredIntraDc :541, xPredIntraAng :592 (wide angles, reference extension, cubic / Gauss /
 *             linear interpolation, angular PDPC), IntraPredSampleFilterCore :212 (PDPC of planar / DC), xPredIntraBDPCM :850;
 *             initIntraMip / predIntraMip :1906,:1919 with PredictorMIP (MatrixIntraPrediction.cpp:67-330: boundary down-sampling,
 *             matrix stage, up-sampling; weights MipData.h);
 *             xGetLumaRecPixels :1403 / xGetLMParameters :1694 / predIntraChromaLM :519 (CCLM, 4:2:0),
 *             as DecCu::predAndReco calls them for an intra TU (DecCu.cpp:316-371).
 * The availability analysis (cs.getCURestricted walks, IntraPrediction.cpp:1098-1130, :1762-1795) stays host code in the flattener and
 * arrives as counts.  CIIP CUs (predBlendIntraCiip :887) are blocks of this list too: planar prediction blended with the inter prediction K2 left
 * in the block.  Not covered (the flattener must refuse them): ISP, palette, ACT, IBC CUs.
 * Blocks of one list are processed in list order; a block may read what earlier blocks of the list wrote.
 * Refused with B200_ERR_PARAM ("intra block record"): a block (or ISP region) that is not inside one CTU (chroma: half the CTU size), and — on the
 * CTU-resident kernel, the one dense lists take — a CTU with more than 3072 records (128*128/16 luma + 2 * 64*64/4 chroma blocks: more than
 * VVC content can hold, so only overlapping records get there).  The one-CTA-per-block kernel accepts such a list; the count is only known on
 * the device, so the picture path reports it from b200_wait_picture, the kernel-level wrappers on return. */
enum { B200_INTRA_PLANAR = 0, B200_INTRA_DC = 1 /* 2..66 angular */, B200_INTRA_BDPCM_HOR = 67, B200_INTRA_BDPCM_VER = 68,
       B200_INTRA_MIP = 69 /* matrix intra prediction: b200_intra_tu::mip = mode index | transposed << 7 */,
       B200_INTRA_LM = 70, B200_INTRA_MDLM_L = 71, B200_INTRA_MDLM_T = 72 /* cross-component linear model (LM_CHROMA_IDX, MDLM_L_IDX, MDLM_T_IDX), chroma only */ };
enum { B200_INTRA_FILTER_REF = 1, B200_INTRA_AVAIL_TL = 2, B200_INTRA_ADD_RESI = 4 /* reconstruct: clip(pred + residual), see b200_intra_reconstruct */,
       B200_INTRA_LM_ABOVE = 8, B200_INTRA_LM_LEFT = 16 /* CCLM: the CU has an above / left neighbour (xGetLumaRecPixels :1461,:1464) */,
       B200_INTRA_LM_COLLOCATED = 32 /* CCLM: sps_chroma_vertical_collocated_flag (SPS::getCclmCollocatedChromaFlag) */,
       B200_INTRA_ISP = 64 /* luma prediction region of an intra-sub-partition CU, see below */ };
/* Intra sub-partitions (ISP: initIntraPatternChTypeISP IntraPrediction.cpp:966, DecCu.cpp:341-371, CU::getISPSplitDim UnitTools.cpp:360).  One luma record per
 * PREDICTION REGION of the CU, in decoding order: a sub-partition, or — vertical splits of 4xN / 8xN CUs, whose sub-partitions are 1 / 2 samples wide — the 4-wide
 * region that holds four / two of them (CU::isPredRegDiffFromTB).  x, y, log2w, log2h: the region; mode: the CU's final luma mode (planar, DC, angular);
 * mip: split (1 horizontal: regions stacked top to bottom, 2 vertical) | region index << 2 | log2(regions of the CU) << 4 — the CU is rebuilt from them;
 * numAbove / numLeft / B200_INTRA_AVAIL_TL: the CU-level neighbourhood (the CU's reference samples are fetched once, for 2W and 2H); lmLeft / lmAbove: the CU
 * has a left / above neighbour CU; ciip: bit i = the i-th transform unit inside the region carries a residual (B200_INTRA_ADD_RESI: any).  A region reads the
 * reconstruction of the region before it, so the records of a CU must follow each other. */
typedef struct b200_intra_tu {
  uint16_t x, y;          /* top-left in the component's plane, samples                                              */
  uint8_t  log2w, log2h;  /* 2..6 (chroma: height may be 2 = log2h 1)                                                */
  uint8_t  comp;          /* 0 Y, 1 Cb, 2 Cr                                                                         */
  uint8_t  mode;          /* PU::getFinalIntraMode (before the wide-angle mapping), or B200_INTRA_BDPCM_*            */
  uint8_t  multiRefIdx;   /* cu.multiRefIdx() for luma (0, 1, 2), 0 for chroma                                       */
  uint8_t  flags;         /* B200_INTRA_FILTER_REF: useFilteredIntraRefSamples (:1301); B200_INTRA_AVAIL_TL: m_neighborSize[0] */
  uint8_t  numAbove;      /* m_neighborSize[1]: available units above + above-right (unit = 4 luma / 2 chroma samples) */
  uint8_t  numLeft;       /* m_neighborSize[2]: available units left + below-left                                    */
  uint8_t  mip;           /* B200_INTRA_MIP: cu.intraDir[luma] (MIP mode index) | cu.mipTransposedFlag() << 7                    */
  uint8_t  lmAbove, lmLeft;/* CCLM: template units (2 chroma samples) xGetLMParameters finds available above(+right) / left(+below) (:1762-1795) */
  uint8_t  ciip;          /* 0, or wIntra = 1..3 of a CIIP CU (predBlendIntraCiip :887): the block's samples hold the inter prediction (K2);
                             K6 stores (wIntra * intra + (4 - wIntra) * inter + 2) >> 2 (then + residual).  mode is planar.          */
} b200_intra_tu;          /* 16 bytes */
/* Kernel-level K6: host planes in (reconstructed neighbourhood), prediction written into the blocks, host planes out.  Both K6 entry points
 * return B200_ERR_PARAM, before any device work and with the planes untouched, for an invalid geometry (b200_geom) and for any record the picture
 * path's validation refuses ("intra block record": geometry, mode, ISP region, or availability reaching outside the picture). */
B200_API int b200_intra_predict(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* tus, size_t numTus);
/* The same with the reconstruction step of DecCu::predAndReco (DecCu.cpp:390-398): blocks flagged B200_INTRA_ADD_RESI store
 * clip(pred + resi[comp][same position]) — what the next block of the list then reads as its reference.  resi planes have the picture's
 * geometry (e.g. the output of b200_k1_residual in mode 1). */
B200_API int b200_intra_reconstruct(const b200_geom* g, int16_t* const planes[3], const int16_t* const resi[3], const b200_intra_tu* tus, size_t numTus);

/* ------------------------------------------------------------------------------------------------
 * Picture level: the DecLibRecon seam (reference DecoderLib/DecLibRecon.h:184-191, .cpp:429 decompressPicture,
 * :684 waitForPrevDecompressedPic).  A context owns the decoded-picture buffer (DPB) in device memory, a ring of
 * work-list arenas and one CUDA stream; pictures are processed in submission order (a picture may reference any
 * slot written by an earlier submission — the stream order replaces the reference's reconDone barriers).
 *   per picture:  H2D work lists -> K2 (prediction into the work plane) -> K1 (residual + reco, in place) ->
 *                 K3 deblock V,H (in place) -> K4 SAO (-> second work plane) -> K5 ALF/CC-ALF (-> DPB slot)
 *   with LMCS:    K2 stores forward-mapped luma -> K1 luma TUs -> K6 luma blocks -> per-VPDU chroma scale (from the reconstructed, mapped luma) ->
 *                 K1 chroma TUs (scaled residual) -> K6 chroma blocks -> inverse luma map -> K3 ...
 *   with intra:   ... K1 (TUs of intra / CIIP CUs leave their residual in residual planes) -> K6 (intra and CIIP blocks in decoding order,
 *                 prediction [blend] + residual) -> K3 ...
 * Samples of tools the device path does not have (ISP, IBC) can be supplied in `given` (whole planes, uploaded before K2); inter PUs,
 * residuals and K6 blocks overwrite/add on top.
 * ---------------------------------------------------------------------------------------------- */
typedef struct b200_ctx b200_ctx;

/* LMCS (luma mapping with chroma scaling), reference CommonLib/Reshape.cpp.  The tables are the members Reshape::constructReshaper
 * (:317-373) derives from the LMCS APS — the glue copies them out of the per-thread Reshape object after initSlice:
 *   forward map of the inter-predicted luma (rspBufFwd :410 -> rspFwdCore, Buffer.cpp:321), fused into K2's luma stores;
 *   chroma residual scaling (calculateChromaAdjVpduNei :192, scaleSignal Buffer.cpp:412) in K1's chroma pass;
 *   inverse map of the reconstructed luma before deblocking (rspCtuBcw :377 -> applyLut with m_invLUT).
 * One record per VPDU (64x64 luma for 128-CTUs, else one per CTU; raster order, ceil(W/size) per row): position of the CU that
 * covers the VPDU's top-left sample (cs.getCU at :217) and whether that CU has a left / above neighbour CU the reference may read
 * (getCURestricted :218-219: inside the picture, same slice and tile). */
typedef struct b200_lmcs_vpdu { uint16_t x, y; uint8_t availLeft, availAbove; } b200_lmcs_vpdu;   /* 6 bytes */
typedef struct b200_lmcs {
  int32_t chromaAdj;              /* ph_chroma_residual_scale_flag (SliceReshapeInfo::enableChromaAdj)                 */
  int32_t minBinIdx, maxBinIdx;   /* reshaperModelMinBinIdx / MaxBinIdx                                                 */
  int32_t orgCW;                  /* m_initCW = (1 << bitDepth) / 16                                                    */
  int16_t reshapePivot[17];       /* m_reshapePivot (LmcsPivot)                                                         */
  int16_t inputPivot[17];         /* m_inputPivot                                                                       */
  int16_t fwdScaleCoef[16];       /* m_fwdScaleCoef                                                                     */
  int32_t chromaAdjHelpLUT[16];   /* m_chromaAdjHelpLUT                                                                 */
  const int16_t* invLUT;          /* m_invLUT, 1 << bitDepth entries                                                    */
  const b200_lmcs_vpdu* vpdus;    /* needed when chromaAdj != 0                                                         */
} b200_lmcs;

typedef struct b200_picture {
  int32_t dstSlot;                       /* DPB slot that receives the final picture                                  */
  int32_t flags;                         /* B200_PIC_*                                                                */
  const int16_t* given[3];               /* optional planes (geometry strides) with pre-reconstructed samples, or NULL */
  const b200_pu* pus; size_t numPus;     /* K2 */
  size_t numDmvr;                        /*     size of the DMVR MV-delta output (entries)                            */
  const b200_tu* tus; size_t numTus;     /* K1 */
  const int16_t* coefs; size_t numCoefs;
  const int32_t* scaling; size_t numScaling;
  const b200_lf_param *lfV, *lfH;        /* K3 (B200_PIC_DEBLOCK) */
  const uint8_t* ctuSlice; const b200_lf_slice* lfSlices; int32_t numLfSlices; const b200_lf_seq* lfSeq;
  const b200_sao_ctu* sao;               /* K4 (B200_PIC_SAO) */
  const b200_vb* vb;
  const b200_alf_ctu* alf;               /* K5 (B200_PIC_ALF) */
  const b200_alf_tables* alfTabs;
  const b200_wp* wp; int32_t numWp;      /* explicit weighted prediction entries referenced by b200_pu::wpIdx, or NULL / 0 */
  const b200_lmcs* lmcs;                 /* B200_PIC_LMCS: every slice of the picture has LMCS on (samples in `given` must already be in the
                                            mapped domain); intra / CIIP blocks are predicted in the mapped domain                               */
  const b200_intra_tu* intraTus;         /* K6: intra blocks of the picture in decoding order, or NULL.  Runs after K2 and K1: blocks read the     */
  size_t numIntraTus;                    /* reconstruction of inter and earlier intra neighbours.  With LMCS chroma scaling: luma blocks, then the
                                            per-VPDU scales, then the chroma blocks (see "with LMCS" above)                                     */
  /* B200_PIC_DERIVE_LF (with B200_PIC_DEBLOCK; lfV and lfH must then be NULL): the records the device derives both grids from (see b200_lf_cu) */
  const b200_lf_cu* lfCus; size_t numLfCus;
  const b200_lf_tu* lfTus; size_t numLfTus;
  const uint32_t* lfCtuCus;              /* [number of CTUs + 1]: index of each CTU's first CU record (raster order), then numLfCus            */
  const uint8_t* lfSliceB;               /* [numLfSlices]: 1 for a B slice (Slice::isInterB, LoopFilter.cpp:1235)                          */
} b200_picture;
enum { B200_PIC_DEBLOCK = 1, B200_PIC_SAO = 2, B200_PIC_ALF = 4, B200_PIC_LMCS = 8, B200_PIC_DERIVE_LF = 16 };

/* create(): reference DecLibRecon::create (DecLibRecon.cpp:392). numSlots = DPB size, numArenas = pictures whose work
 * lists may be resident at once (>= 2 for upload/compute overlap). device < 0: current device.  Returns B200_ERR_PARAM for an
 * invalid geometry (b200_geom). */
B200_API int  b200_ctx_create(b200_ctx** ctx, const b200_geom* g, int numSlots, int numArenas, int device);
B200_API void b200_ctx_destroy(b200_ctx* ctx);
/* Host planes -> DPB slot (e.g. an IRAP picture reconstructed elsewhere, or test content). Synchronous; waits for pending asynchronous outputs of the
 * slot's buffer before it overwrites it. */
B200_API int  b200_ctx_load_slot(b200_ctx* ctx, int slot, const int16_t* const planes[3]);
/* decompressPicture() = b200_pic_upload + b200_pic_run.  Returns the arena handle (>= 0) or a negative error.
 *
 * b200_pic_upload: non-blocking, no per-record host work.  The caller's arrays are copied as they are to the next arena (async H2D on
 *   the context's upload stream: pass pinned memory, see b200_host_register); two small kernels validate the PU / TU records and sort
 *   their indices into the work lists of the compute kernels on the device.  Its only host checks are O(1): with SAO or ALF on it returns
 *   B200_ERR_PARAM for the geometry, ALF table counts and virtual boundaries b200_sao_picture / b200_alf_picture refuse.
 * b200_pic_run: enqueues the picture's kernel chain.  It sizes the grids from the list lengths the upload produced, so it waits (host)
 *   until that upload has finished; a caller that uploads picture n+1 before it runs picture n (a parser running ahead of
 *   reconstruction) never waits.  Once it returns the picture's upload is complete: the caller may overwrite or free the host arrays.  An invalid record (reference slot outside the DPB, impossible block size, BDOF/DMVR on a block that
 *   cannot have it, DMVR at more than 10 bit) makes it return B200_ERR_PARAM without running anything.
 * A handle may be run several times (device-resident benchmarking); it keeps its work lists until its arena is uploaded again (numArenas uploads
 * later), and that upload waits on the device for the kernels of the handle's last run. */
B200_API int  b200_decompress_picture(b200_ctx* ctx, const b200_picture* pic);
B200_API int  b200_pic_upload(b200_ctx* ctx, const b200_picture* pic);            /* -> arena handle */
B200_API int  b200_pic_run(b200_ctx* ctx, int arena);
/* waitForPrevDecompressedPic(): blocks until every picture submitted so far is final; copies the DMVR MV deltas of
 * `arena` (needed by the CPU's TaskFinishMotionInfo, DecCu.cpp:161) to dmvrMv (may be NULL).  Returns B200_ERR_PARAM when K6 refused the
 * arena's intra list on the device (more than 3072 records in one CTU, see b200_intra_tu) or an intra block waited for a neighbour that never
 * finished; the picture's samples are then undefined, the context stays usable. */
B200_API int  b200_wait_picture(b200_ctx* ctx, int arena, int32_t* dmvrMv, size_t numDmvr);
/* Output: DPB slot -> host planes (vvdec_frame planes; xAddPicture vvdecimpl.cpp:957). Synchronous D2H. */
B200_API int  b200_get_frame(b200_ctx* ctx, int slot, int16_t* const planes[3]);
/* The same two transfers for host planes with margins (vvdec's PelStorage, Buffer.cpp:645: stride > width), strides in samples:
 * reference pictures reconstructed by the CPU back end enter the device DPB, finished pictures land in Picture::m_bufs. */
B200_API int  b200_ctx_load_slot_strided(b200_ctx* ctx, int slot, const int16_t* const planes[3], const ptrdiff_t strides[3]);
B200_API int  b200_get_frame_strided(b200_ctx* ctx, int slot, int16_t* const planes[3], const ptrdiff_t strides[3]);
/* Asynchronous output: the D2H copy runs on a second stream after the picture is final and overlaps the next pictures' kernels;
 * the context makes later pictures (and b200_ctx_load_slot*) wait before they overwrite a buffer that is still being read — by every pending
 * reader, whichever output call and stream it came from (two readers on different streams: the later one's stream first waits for the earlier
 * one).  Returns a ticket (>= 0);
 * b200_frame_wait(ticket) blocks until those planes are complete in host memory (pinned memory recommended). */
B200_API int  b200_get_frame_async(b200_ctx* ctx, int slot, int16_t* const planes[3]);
B200_API int  b200_frame_wait(b200_ctx* ctx, int ticket);
/* Device-resident output for the multi-GPU gather (SURVEY 8e): the frame is copied device to device into planesDev[] (geometry strides) on the CUDA
 * stream the caller passes (cudaStream_t as void*; e.g. the stream NCCL sends from): that stream first waits for every picture submitted so far. */
B200_API int  b200_get_frame_device_async(b200_ctx* ctx, int slot, int16_t* const planesDev[3], void* cudaStream);
/* Output formats of the application layer, converted on the device before the D2H copy (SURVEY 8f-3):
 *   B200_OUT_16    int16 planes, stride = geometry stride (what vvdecFrame carries for bit depths > 8)
 *   B200_OUT_PYUV  4 samples in 5 bytes, rows back to back, W*5/4 bytes per row — the `.pyuv` / --pyuv writer of vvdecapp
 *                  (App/vvdecapp/vvdecHelper.h:106-150); 10-bit only, width divisible by 8 (vvdecapp.cpp:1179)
 *   B200_OUT_8     one byte per sample, sample >> (bitDepth - 8), rows back to back (vvdecHelper.h:75-104)
 * planes[c] must hold b200_frame_bytes(g, fmt, c) bytes.  Returns a ticket for b200_frame_wait, like b200_get_frame_async. */
enum { B200_OUT_16 = 0, B200_OUT_PYUV = 1, B200_OUT_8 = 2 };
B200_API size_t b200_frame_bytes(const b200_geom* g, int fmt, int comp);
B200_API int  b200_get_frame_fmt_async(b200_ctx* ctx, int slot, int fmt, void* const planes[3]);
/* Film grain synthesis on the output frame (SURVEY 8f-3): the per-sample part of the reference's VFGS model,
 *   replaces  FilmGrainImpl::add_grain_block / make_grain_pattern / scale_and_output (FilmGrain/FilmGrainImpl.cpp:129,:198,:247 and their
 *             SSE4.1/AVX2 versions FilmGrainImpl_X86_SIMD.h), driven per line by FilmGrain::add_grain_line (FilmGrain.cpp:836) from
 *             VVDecImpl::xAddGrain (vvdec/vvdecimpl.cpp:898; 16-line tasks on the decoder's thread pool).
 * The tables are what FilmGrain::updateFGC -> init_sei (FilmGrain.cpp:560,:730 — host code, once per SEI) leaves in FilmGrainImpl, the
 * line seeds what FilmGrain::prepareBlockSeeds (:794) produces for this frame.  The DPB picture is not modified (it may still be
 * referenced): grain is added on the way out.  8 and 10 bit, 4:2:0 / 4:0:0 (FilmGrainImpl::set_depth :357). */
typedef struct b200_film_grain {
  const int8_t*   pattern;       /* [2][8][64][64]  FilmGrainImpl::pattern[luma|chroma][0..7]; chroma uses the top-left 32x32 of each      */
  const uint8_t*  sLUT;          /* [3][256]        FilmGrainImpl::sLUT  (scale by 8-bit intensity)                                         */
  const uint8_t*  pLUT;          /* [3][256]        FilmGrainImpl::pLUT  (pattern index << 4 by intensity; index < 8)                       */
  const uint32_t* lineSeeds;     /* [(height+15)/16] FilmGrain::m_line_seeds                                                                */
  uint8_t         scaleShift;    /* FilmGrainImpl::scale_shift after set_depth / set_scale_shift; scaleShift + bitDepth - 8 in 8..13       */
  uint8_t         compPresent[3];/* fgs.comp_model_present_flag                                                                            */
} b200_film_grain;
/* Like b200_get_frame_fmt_async, with grain added before the format conversion.  The arrays are copied (into pinned memory of the context) before
 * the call returns: the caller may overwrite them at once. */
B200_API int  b200_get_frame_grain_async(b200_ctx* ctx, int slot, int fmt, void* const planes[3], const b200_film_grain* fg);
/* Decoded-picture hash computed on the device (SURVEY 8f-3): what calcCRC / calcChecksum (CommonLib/PicYuvMD5.cpp:138,:179) produce for
 * the decoded picture hash SEI check (calcAndPrintHashStatus :261), so a verify-only run reads back 6 / 12 bytes instead of the frame.
 * method uses the vvdecHashType values (vvdec/sei.h): 1 CRC (2 bytes per component), 2 checksum (4 bytes per component); the digest bytes
 * are in PictureHash::hash order (Y, Cb, Cr).  MD5 (0) is one serial chain per plane and returns B200_ERR_UNSUPPORTED.
 * digest must hold 12 bytes (pinned memory recommended).  Returns a ticket for b200_frame_wait. */
enum { B200_HASH_MD5 = 0, B200_HASH_CRC = 1, B200_HASH_CHECKSUM = 2 };
B200_API int  b200_frame_hash_async(b200_ctx* ctx, int slot, int method, uint8_t* digest);
/* Timing helpers for bench.py: CUDA events on the context stream. */
B200_API int  b200_ctx_mark(b200_ctx* ctx, int which /*0 start, 1 stop*/);
B200_API int  b200_ctx_elapsed_ms(b200_ctx* ctx, float* ms);
B200_API long long b200_ctx_kernel_launches(b200_ctx* ctx);
/* Per-kernel-family device time (CUDA events on the context stream around each family's launches of b200_pic_run).
 * Families: 0 K2 translational tiles, 1 K2 affine tiles, 2 K1, 3 K3 vertical, 4 K3 horizontal, 5 K4, 6 K5 luma, 7 K5 chroma.
 * set_profiling(1) enables event recording (adds a few us per picture); get_kernel_ms sums and resets the collected times. */
enum { B200_KF_MC_TILE = 0, B200_KF_MC_AFFINE, B200_KF_K1, B200_KF_LF_V, B200_KF_LF_H, B200_KF_SAO, B200_KF_ALF_LUMA, B200_KF_ALF_CHROMA,
       B200_KF_INTRA /* K6 incl. its ordering pre-passes */, B200_KF_LMCS /* per-VPDU scale + inverse map */,
       B200_KF_LF_DERIVE /* B200_PIC_DERIVE_LF: CU maps, motion field, edge grids */, B200_KF_COUNT };
B200_API int  b200_ctx_set_profiling(b200_ctx* ctx, int on);
B200_API int  b200_ctx_get_kernel_ms(b200_ctx* ctx, float ms[8], int counts[8]);          /* the first eight families */
B200_API int  b200_ctx_get_kernel_ms_n(b200_ctx* ctx, float* ms, int* counts, int n);     /* n <= B200_KF_COUNT families */
/* Pin / unpin caller-owned host memory (cudaHostRegister) so that the H2D / D2H copies of the picture-level calls are asynchronous. */
B200_API int  b200_host_register(void* ptr, size_t bytes);
B200_API int  b200_host_unregister(void* ptr);

#ifdef __cplusplus
}
#endif
#endif
