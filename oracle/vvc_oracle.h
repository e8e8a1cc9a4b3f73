/* vvc_oracle.h — CPU restatement ("oracle") of the VVdeC pixel-reconstruction hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may call it.
 * The product path (vvdec_b200/csrc) never links or falls back to this code.
 *
 * Parity status: PINNED.  Every function here is checked bit-for-bit against the reference's own
 * scalar *Core functions compiled from the reference sources into oracle/_ref/libvvdec_ref.so
 * (oracle/Makefile.ref, oracle/ref_shim.cpp; tests/test_oracle_vs_ref.py), and against the golden
 * vectors under tests/golden/ that were generated from that library (tools/make_golden.py).
 *
 * Plain C99, scalar, single-threaded.  Each function cites the reference file:line it restates
 * (paths relative to vvdec source/Lib/CommonLib unless noted).
 */
#ifndef VVC_ORACLE_H
#define VVC_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#include "../include/vvdec_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- K1 building blocks -------------------------------------------------------------------- */
/* Quant.cpp:122-179 DeQuantImpl (UseScalingList = sl != NULL); q is int16 levels with stride qStride. */
void orc_dequant(int width, int maxX, int maxY, int scale, const int32_t* sl, const int16_t* q, size_t qStride,
                 int32_t* coef, int rightShift, int inputMaximum, int32_t transformMaximum);
/* same, 32-bit levels (DeQuantPCM, Quant.cpp:208: BDPCM path dequantises the accumulated block in place) */
void orc_dequant32(int width, int maxX, int maxY, int scale, const int32_t* sl, const int32_t* q, size_t qStride,
                   int32_t* coef, int rightShift, int inputMaximum, int32_t transformMaximum);
/* TrQuant.cpp:79-106 invLfnstNxNCore. */
void orc_inv_lfnst(const int32_t* src, int32_t* dst, unsigned set, unsigned index, unsigned size, int zeroOutSize);
/* TrQuant_EMT.cpp:103-121 _fastInverseMM / :126-354 fastInverse{DCT2,DCT8,DST7}_B{2..64}: one 1-D stage. */
void orc_inv_1d(int trType, int n, const int32_t* src, int32_t* dst, int shift, int line, int skipLine, int skipLine2,
                int clip, int32_t outMin, int32_t outMax);
/* TrQuant_EMT.cpp:366 cpyResiClipCore. */
void orc_cpy_resi_clip(const int32_t* src, int16_t* dst, ptrdiff_t stride, unsigned w, unsigned h,
                       int32_t outMin, int32_t outMax, int32_t round, int32_t shift);
/* TrQuant.cpp:290 invTransformNxN for one record (dequant → LFNST → xIT | TS), residual to resi[stride]. */
void orc_tu_residual(const b200_tu* tu, int bitDepth, const int16_t* coefs, const int32_t* scaling,
                     int16_t* resi, ptrdiff_t stride);
/* DecCu.cpp:536 reconstructResi over a list + (mode 0) the pred+resi clip of Buffer.cpp:83 recoCore. */
void orc_k1_residual(const b200_geom* g, int16_t* const planes[3], const b200_tu* tus, size_t numTus,
                     const int16_t* coefs, const int32_t* scaling, int mode);

/* ---- LMCS (Reshape.cpp) ------------------------------------------------------------------------- */
/* Buffer.cpp:321 rspFwdCore on a w x h block (the luma prediction of one inter CU, DecCu.cpp:460-474). */
void orc_lmcs_fwd_block(int16_t* ptr, ptrdiff_t stride, int w, int h, int bitDepth, const b200_lmcs* L);
/* rspBufFwd over the luma area of every PU of a list. */
void orc_lmcs_fwd_pus(const b200_geom* g, int16_t* luma, const b200_pu* pus, size_t numPus, const b200_lmcs* L);
/* Reshape.cpp:192 calculateChromaAdjVpduNei for VPDU record v (averages the mapped-domain luma left of / above the CU at (v.x,v.y)). */
int orc_lmcs_vpdu_scale(const b200_geom* g, const int16_t* luma, const b200_lmcs* L, const b200_lmcs_vpdu* v);
/* Buffer.cpp:412 scaleSignal on one residual sample. */
int orc_lmcs_scale_resi(int r, int scale, int bitDepth);
/* DecCu.cpp:483 finishLMCSAndReco order for an all-inter picture: luma TUs (reco), chroma scale per VPDU, chroma TUs (scaled residual, reco). */
void orc_k1_residual_lmcs(const b200_geom* g, int16_t* const planes[3], const b200_tu* tus, size_t numTus,
                          const int16_t* coefs, const int32_t* scaling, const b200_lmcs* L);
/* Reshape.cpp:377 rspCtuBcw over the whole luma plane (Buffer.cpp:200 applyLutCore). */
void orc_lmcs_inv_plane(const b200_geom* g, int16_t* luma, const b200_lmcs* L);

/* ---- output formats (App/vvdecapp/vvdecHelper.h:63 _writeComponentToFile) ---------------------------------------- */
/* :115-128 packed yuv: 4 samples -> 5 bytes per group, rows back to back (w * 5 / 4 bytes). */
void orc_pack_pyuv(const int16_t* src, ptrdiff_t stride, int w, int h, uint8_t* dst);
/* :86-93 8-bit narrowing (the writer's >> 2 for 10 bit; >> (bitDepth - 8) in general). */
void orc_narrow8(const int16_t* src, ptrdiff_t stride, int w, int h, int bitDepth, uint8_t* dst);
/* decoded-picture hash of one plane: method 1 CRC (2 bytes), 2 checksum (4 bytes); returns the digest length */
/* K6 intra prediction of regular modes (k8_intra.c): blocks in list order, prediction written into the planes */
void orc_intra_tu(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* t);
void orc_intra_predict(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* tus, size_t numTus);
/* intra sub-partitions of one luma CU (groundwork for the next K6 slice; see k8_intra.c) */
void orc_intra_isp_cu(const b200_geom* g, int16_t* luma, const int16_t* resi, int x0, int y0, int w, int h, int ispMode, int dirMode,
                      int availTL, int numAbove, int numLeft, int leftAvail, int aboveAvail, unsigned resiMask);
void orc_intra_reconstruct(const b200_geom* g, int16_t* const planes[3], const int16_t* const resi[3], const b200_intra_tu* tus, size_t numTus);
/* CCLM parameter derivation of one chroma record (xGetLMParameters): a, b, shift; the min / max luma and chroma averages; the four (luma, chroma)
 * template pairs the min / max grouping sees (selL / selC, after the two-sample path duplicates its pair), cntT / cntL of them from the above / left
 * template; normDiff (-1 without a slope) and whether shift < 1 clamped the slope; blkMin / blkMax: the range of the block's down-sampled luma.  Reads the planes as orc_intra_tu would at that point of a list. */
typedef struct orc_cclm { int32_t a, b, shift, minL, maxL, minC, maxC, cntT, cntL, normDiff, clamped, selL[4], selC[4], blkMin, blkMax; } orc_cclm;
void orc_cclm_params(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* t, orc_cclm* out);
/* What the prediction of one regular intra record went through.  Each xxxMin / xxxMax pair is the range of the values a clip site saw before it clipped
 * (INT32_MAX / INT32_MIN where the record never reached it): cubic: the 4-tap cubic interpolation of a fractional luma angle; pdpc: PDPC of the
 * horizontal / vertical modes; mip: the reduced MIP prediction; reco: pred + resi; pred: the final prediction (before the residual).  subst: the
 * values reference substitution wrote (1 << (bitDepth - 1) without any neighbour, else the padding copied from available samples).  filtered: the
 * [1 2 1] filtered reference was used; interp: 0 none, 1 cubic, 2 Gaussian (luma), 3 two-tap linear (chroma); mipSizeId (-1: not MIP),
 * mipInputOffset (the first down-sampled boundary sample) and mipInput0 (the first matrix input after the rebase). */
typedef struct orc_intra_trace {
  int32_t substMin, substMax, cubicMin, cubicMax, pdpcMin, pdpcMax, mipMin, mipMax, recoMin, recoMax, predMin, predMax;
  int32_t filtered, interp, mipSizeId, mipInputOffset, mipInput0;
} orc_intra_trace;
/* one record as orc_intra_reconstruct runs it (prediction, then pred + resi where the record adds a residual and resi is not NULL): the planes advance */
void orc_intra_probe(const b200_geom* g, int16_t* const planes[3], const int16_t* const resi[3], const b200_intra_tu* t, orc_intra_trace* out);
/* film grain synthesis, per-sample part (FilmGrainImpl::add_grain_block); tables as FilmGrainImpl holds them after FilmGrain::updateFGC:
 * pattern [2][8][64][64], sLUT / pLUT [3][256], lineSeeds [(h+15)/16] (FilmGrain::prepareBlockSeeds); 4:2:0, planes in place */
void orc_film_grain(int16_t* const planes[3], const ptrdiff_t strides[3], int w, int h, int bitDepth, const int8_t* pattern, const uint8_t* sLUT,
                    const uint8_t* pLUT, const uint32_t* lineSeeds, int scaleShift, const uint8_t compPresent[3]);
int orc_plane_hash(int method, int bitDepth, const int16_t* src, ptrdiff_t stride, int w, int h, uint8_t* digest);

/* ---- K3 deblocking -------------------------------------------------------------------------- */
/* LoopFilter.cpp:213 xPelFilterLumaCore (4 lines). */
void orc_lf_pel_filter_luma(int16_t* src, ptrdiff_t step, ptrdiff_t offset, int tc, int sw, int thrCut,
                            int filterSecondP, int filterSecondQ, int bitDepth);
/* LoopFilter.cpp:129 xFilteringPandQCore (4 lines). */
void orc_lf_filtering_pq(int16_t* src, ptrdiff_t step, ptrdiff_t offset, int numP, int numQ, int tc);
/* LoopFilter.cpp:375 loopFilterCTU over the whole picture: dirs bit0 = all vertical edges, bit1 = all horizontal. */
void orc_lf_deblock(const b200_geom* g, int16_t* const planes[3], const b200_lf_param* lfV, const b200_lf_param* lfH,
                    const uint8_t* ctuSlice, const b200_lf_slice* slices, const b200_lf_seq* seq, int dirs);

/* ---- K4 SAO ---------------------------------------------------------------------------------- */
/* SampleAdaptiveOffset.cpp:64 offsetBlock_core for one CTU component (same argument meaning; vb = positions relative to the block). */
void orc_sao_offset_block(int bitDepth, int typeIdx, const int* offset /*32*/, const int16_t* src, int16_t* dst,
                          ptrdiff_t srcStride, ptrdiff_t dstStride, int width, int height, unsigned avail,
                          int numVerVb, const int* verVb, int numHorVb, const int* horVb);
/* SAOProcessCTU over the picture (SampleAdaptiveOffset.cpp:522,:661). dst must be pre-filled by the caller? No: it copies src first. */
void orc_sao_picture(const b200_geom* g, const int16_t* const src[3], int16_t* const dst[3], const b200_sao_ctu* ctus, const b200_vb* vb);

/* ---- K5 ALF ---------------------------------------------------------------------------------- */
/* AdaptiveLoopFilter.cpp:969 deriveClassificationBlk: cls[(i/4)*8 + j/4] = classIdx | transposeIdx<<8 for the blk (<=32x32). */
void orc_alf_classify(uint16_t* cls, const int16_t* srcLuma, ptrdiff_t stride, int blkX, int blkY, int blkW, int blkH,
                      int shift, int vbCtuHeight, int vbPos);
/* AdaptiveLoopFilter.cpp:1175 filterBlk<7>/<5>: cls may be NULL for chroma (5x5). src/dst are plane origins. */
void orc_alf_filter_blk(int is7x7, const uint16_t* cls, int16_t* dst, ptrdiff_t dstStride, const int16_t* src, ptrdiff_t srcStride,
                        int blkX, int blkY, int blkW, int blkH, const int16_t* coeff, const int16_t* clip, int bitDepth,
                        int vbCtuHeight, int vbPos);
/* AdaptiveLoopFilter.cpp:1348 filterBlkCcAlf (4:2:0). */
void orc_alf_ccalf_blk(int16_t* dstChroma, ptrdiff_t chromaStride, const int16_t* srcLuma, ptrdiff_t lumaStride,
                       int cX, int cY, int cW, int cH, const int16_t* coeff, int bitDepth, int vbCtuHeight, int vbPos);
/* processCTU over the picture, !isCrssByVBs path (AdaptiveLoopFilter.cpp:466,:664-741); src planes are read with
 * coordinates clamped to the picture (== prepareCTU's border extension, :453). */
void orc_alf_picture(const b200_geom* g, const int16_t* const src[3], int16_t* const dst[3], const b200_alf_ctu* ctus,
                     const b200_alf_tables* tabs);

/* ---- K2 inter prediction --------------------------------------------------------------------- */
/* InterPrediction.cpp:1372 motionCompensation for a list of PUs (regular uni/bi, BCW, BDOF, DMVR, affine + PROF).
 * refs[slot*3+comp]; reference samples outside the picture are read with clamped coordinates (== border extension). */
void orc_mc_predict(const b200_geom* g, int16_t* const dst[3], const int16_t* const* refs, const b200_pu* pus, size_t numPus, int32_t* dmvrMv);
/* the same with explicit weighted prediction (WeightPrediction.cpp:164 addWeightBi, :238 addWeightUni) for PUs with wpIdx != 0 */
void orc_mc_predict_wp(const b200_geom* g, int16_t* const dst[3], const int16_t* const* refs, const b200_pu* pus, size_t numPus, int32_t* dmvrMv, const b200_wp* wp);

#ifdef __cplusplus
}
#endif
/* LMCS together with intra / CIIP blocks (k6_lmcs.c) */
void orc_lmcs_vpdu_scales(const b200_geom* g, const int16_t* luma, const b200_lmcs* L, int32_t* scale);
void orc_k1_residual_sel(const b200_geom* g, int16_t* const planes[3], int16_t* const resi[3], const b200_tu* tus, size_t numTus,
                         const int16_t* coefs, const int32_t* scaling, int compSel, const int32_t* scale);
#endif
