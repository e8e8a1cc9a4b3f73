// rules.cuh — what a geometry and every kind of record must satisfy before a kernel may use it, stated once.  The kernel-level wrappers (api.cu) check
// each record on the host with these functions before any device work; the picture path (picture.cu) checks its O(1) inputs on the host and its
// records on the device (bucket.cu, k6_intra.cu, lmcs.cu), where a failure raises one error bit per list.  Each function returns nullptr for a legal input, or
// a short reason: the host prints it after the entry point's name, the device only tests it for null.
#pragma once
#include <stdint.h>
#include <vector>
#include "../../include/vvdec_b200.h"

namespace b200 {

// 4:0:0 or 4:2:0, CTU 32 / 64 / 128, bit depth 8..maxBitDepth, a picture of whole 8x8 units, every present plane's stride at least its width and a
// multiple of strideAlign (K4 and K5 move 4 samples per 8-byte access, Cr included)
__host__ __device__ inline const char* geom_problem(const b200_geom& g, int maxBitDepth, int strideAlign)
{
  if (g.chromaFormat != 0 && g.chromaFormat != 1) return "geometry: chromaFormat (only 0 = 4:0:0 and 1 = 4:2:0)";
  if (g.ctuSize != 32 && g.ctuSize != 64 && g.ctuSize != 128) return "geometry: CTU size (32, 64 or 128)";
  if (g.bitDepth < 8 || g.bitDepth > maxBitDepth) return maxBitDepth == 10 ? "geometry: bit depth (8..10)" : "geometry: bit depth (8..12)";
  if (g.width <= 0 || g.height <= 0 || (g.width & 7) || (g.height & 7)) return "geometry: picture size is not a multiple of 8";
  for (int c = 0; c < (g.chromaFormat ? 3 : 1); c++) {
    if (g.stride[c] < (c ? g.width >> 1 : g.width)) return "geometry: a plane stride is smaller than the plane's width";
    if (g.stride[c] % strideAlign) return "geometry: a plane stride is not a multiple of 4 samples";
  }
  return nullptr;
}
// log2 of the CTU size of a geometry geom_problem accepts
__host__ __device__ inline int ctu_log2(const b200_geom& g) { return g.ctuSize == 128 ? 7 : g.ctuSize == 64 ? 6 : 5; }

// ---- K2: PU records (b200_pu) ----
struct PuLimits { int numSlots, bitDepth, numWp, W, H; unsigned numDmvr; };
inline PuLimits pu_limits(const b200_geom& g, int numSlots, int numWp, size_t numDmvr)
{
  PuLimits l; l.numSlots = numSlots; l.bitDepth = g.bitDepth; l.numWp = numWp; l.W = g.width; l.H = g.height;
  l.numDmvr = (unsigned)(numDmvr > 0xffffffffu ? 0xffffffffu : numDmvr);
  return l;
}
__host__ __device__ inline const char* pu_problem(const b200_pu& p, const PuLimits& lim)
{
  const int s0 = p.refSlot[0], s1 = p.refSlot[1], w = p.w, h = p.h, f = p.flags;
  const bool bi = s0 >= 0 && s1 >= 0, aff = f & B200_PU_AFFINE;
  if (s0 >= lim.numSlots || s1 >= lim.numSlots || (s0 < 0 && s1 < 0)) return "invalid reference slots";
  // sides are multiples of 4 (CUs: powers of two; SbTMVP runs: multiples of 8) whose 16-sample tiles end in a 4, 8 or 16 piece: mc_tile maps threads to
  // samples with tw - 1 masks and log2(tw) shifts, so a 12-sample piece (sides 12, 28, 44, ...) would filter wrong columns and store below the tile
  if (w < 4 || h < 4 || w > 128 || h > 128 || (w & 3) || (h & 3) || (w & 15) == 12 || (h & 15) == 12) return "block size";
  // the block must lie inside the picture on the 4x4 grid (kernels write every sample of it), DMVR deltas inside the output array
  if ((p.x & 3) || (p.y & 3) || p.x + w > lim.W || p.y + h > lim.H) return "block outside the picture or off the 4x4 grid";
  if ((f & B200_PU_DMVR) && (unsigned long long)p.dmvrOff + (unsigned)((w < 16 ? 1 : w >> 4) * (h < 16 ? 1 : h >> 4)) > lim.numDmvr) return "DMVR entries past numDmvr";
  // BDOF / DMVR blocks are at least 8x8 with 128 samples (conditions at InterPrediction.cpp:1372-1420); DMVR also needs both lists and
  // is never affine.  A BDOF flag on a uni-predicted or affine PU is ignored, as the launch-side classification always did.
  const bool big = w >= 8 && h >= 8 && w * h >= 128;
  if ((f & B200_PU_DMVR) && (!bi || !big || aff)) return "DMVR on a uni-predicted, affine or small block";
  if ((f & B200_PU_BDOF) && bi && !aff && !big) return "BDOF on a small block";
  if ((f & B200_PU_DMVR) && lim.bitDepth > 10) return "DMVR needs bit depth <= 10 (as the reference)";
  // GEO (InterPrediction.cpp:1461): two partitions = both 'lists' set, 8..64 luma samples per side, never with another tool; bcwW1 = split direction
  if (f & B200_PU_GEO) {
    if (!bi || w < 8 || h < 8 || w > 64 || h > 64 || (w & (w - 1)) || (h & (h - 1)) || (f & (B200_PU_DMVR | B200_PU_BDOF | B200_PU_AFFINE)) || p.wpIdx || (uint8_t)p.bcwW1 > 63)
      return "GEO block";
  // explicit weights: the entry must exist; the reference never combines them with BDOF / DMVR / BCW (InterPrediction.cpp:733, :1406-1420)
  } else if (p.wpIdx && (p.wpIdx > lim.numWp || (f & B200_PU_DMVR) || ((f & B200_PU_BDOF) && bi && !aff) || p.bcwW1 != 4)) return "explicit weights";
  return nullptr;
}

// ---- K1: TU records (b200_tu) ----
struct TuLimits { int W, H, chroma; unsigned numCoefs, numScaling; };
inline TuLimits tu_limits(const b200_geom& g, size_t numCoefs, size_t numScaling)
{
  TuLimits l; l.W = g.width; l.H = g.height; l.chroma = g.chromaFormat != 0;
  l.numCoefs = (unsigned)(numCoefs > 0xffffffffu ? 0xffffffffu : numCoefs); l.numScaling = (unsigned)(numScaling > 0xffffffffu ? 0xffffffffu : numScaling);
  return l;
}
__host__ __device__ inline const char* tu_problem(const b200_tu& t, const TuLimits& lim)
{
  const int l2w = t.log2w, l2h = t.log2h, m = l2w > l2h ? l2w : l2h;
  if (m > 6 || t.comp >= 3) return "size or component";
  // one-sample-wide / -high blocks exist only as luma sub-partitions of an ISP CU (4xN, N >= 16 and the transpose): regular transform, no LFNST
  if ((l2w == 0 || l2h == 0) && (t.comp != 0 || m < 4 || l2w == l2h || t.lfnst || t.ict || (t.flags & (B200_TU_TS | B200_TU_BDPCM_H | B200_TU_BDPCM_V)))) return "thin block outside a luma ISP sub-partition";
  // inside its plane (the joint-CbCr partner plane has the same geometry), level corner and scaling table inside their arrays
  const int w = 1 << l2w, h = 1 << l2h, pw = t.comp ? lim.W >> 1 : lim.W, ph = t.comp ? lim.H >> 1 : lim.H;
  const bool ts = t.flags & B200_TU_TS, bdpcm = t.flags & (B200_TU_BDPCM_H | B200_TU_BDPCM_V);
  if ((t.comp && !lim.chroma) || t.x + w > pw || t.y + h > ph) return "block outside its plane";
  if (t.maxX >= w || t.maxY >= h || (!ts && (t.maxX >= 32 || t.maxY >= 32))) return "level corner outside the block";
  if ((unsigned long long)t.coefOff + (unsigned)((t.maxX + 1) * (t.maxY + 1)) > lim.numCoefs) return "levels past numCoefs";
  if ((t.flags & B200_TU_SCALING) && (unsigned long long)t.slOff + (unsigned)(w * h) > lim.numScaling) return "scaling factors past numScaling";
  if (t.inBits < 1 || t.inBits > 32 || t.rightShift < -31 || t.rightShift > 31) return "dequantisation range";
  // transform skip / BDPCM blocks are at most 32 wide (sps log2MaxTransformSkipBlockSize <= 5): K1 keeps them in the 32x32 working set of their class;
  // BDPCM accumulates over the whole block, so its level corner is the block
  if ((ts || bdpcm) && (w > 32 || h > 32)) return "transform skip / BDPCM block above 32";
  if (bdpcm && (!ts || t.maxX != w - 1 || t.maxY != h - 1 || (t.flags & (B200_TU_BDPCM_H | B200_TU_BDPCM_V)) == (B200_TU_BDPCM_H | B200_TU_BDPCM_V))) return "BDPCM block";
  // LFNST: index 1 or 2, no stray bits, at least 4x4, never with transform skip (the kernel indexes kLfnst* with it)
  if (t.lfnst && ((t.lfnst & 3) < 1 || (t.lfnst & 3) > 2 || (t.lfnst & 0xe0) || ts || w < 4 || h < 4)) return "LFNST";
  // joint CbCr writes the partner chroma plane at the same position
  if (t.ict && (t.comp == 0 || !lim.chroma || t.ict < -3 || t.ict > 3)) return "joint CbCr";
  return nullptr;
}

// ---- K6: intra block records (b200_intra_tu): everything K6 uses as an address ----
// prev = the record before t in the list (null for the first): the region before an ISP region must be the record before it
__host__ __device__ inline const char* intra_problem(const b200_intra_tu& t, const b200_intra_tu* prev, const b200_geom& g)
{
  const int W = g.width, H = g.height, w = 1 << t.log2w, h = 1 << t.log2h;
  if (t.flags & B200_INTRA_ISP) {                             // ISP region record (B200_INTRA_ISP, include/vvdec_b200.h)
    const int sp = t.mip & 3, k = (t.mip >> 2) & 3, l2n = (t.mip >> 4) & 3, nReg = 1 << l2n;
    if (t.comp || t.mode > 66 || t.multiRefIdx || (sp != 1 && sp != 2) || l2n > 2 || (l2n == 0 && (sp != 2 || w != 4)) /* one region: a 4-wide CU split into 1- or 2-sample columns */ || k >= nReg || (t.mip >> 6) || t.log2w < 2 || t.log2w > 6 || t.log2h > 6)
      return "bad ISP region";
    const int cw = sp == 2 ? w * nReg : w, ch = sp == 1 ? h * nReg : h, cx = t.x - (sp == 2 ? k * w : 0), cy = t.y - (sp == 1 ? k * h : 0);
    if (cw > 64 || ch > 64 || ch < 4 || cw * ch < 32 || cx < 0 || cy < 0 || (cx & 3) || (cy & 3) || cx + cw > W || cy + ch > H) return "bad ISP region";
    if (t.numAbove > 2 * cw / 4 || t.numLeft > 2 * ch / 4 || (t.numAbove && !cy) || (t.numLeft && !cx) || ((t.flags & B200_INTRA_AVAIL_TL) && (!cx || !cy))
        || cx + (int)t.numAbove * 4 > W || cy + (int)t.numLeft * 4 > H || (t.lmLeft && !cx) || (t.lmAbove && !cy)) return "bad ISP region";
    if (k && (!prev || !(prev->flags & B200_INTRA_ISP) || prev->mip != (uint8_t)(t.mip - 4) || prev->log2w != t.log2w || prev->log2h != t.log2h || prev->mode != t.mode
              || prev->x != t.x - (sp == 2 ? w : 0) || prev->y != t.y - (sp == 1 ? h : 0))) return "bad ISP region (the region before it is not the record before it)";
  } else {
    const int pw = t.comp ? W >> 1 : W, ph = t.comp ? H >> 1 : H, unit = t.comp ? 2 : 4;
    if (!(t.comp < (g.chromaFormat ? 3 : 1) && t.log2w >= 2 && t.log2w <= 6 && t.log2h >= 1 && t.log2h <= 6 && t.x + w <= pw && t.y + h <= ph && !(t.x % unit) && !(t.y % unit)))
      return "bad geometry";
  }
  // the CTU-resident kernel addresses its tile by the CTU of the block's top-left sample (chroma: CTU size halved), so a block (or ISP region) reaching
  // into the next CTU would write outside its tile rows
  const int cl = ctu_log2(g) - (t.comp ? 1 : 0);
  if ((t.x >> cl) != ((t.x + w - 1) >> cl) || (t.y >> cl) != ((t.y + h - 1) >> cl)) return "not inside one CTU";
  if (t.flags & B200_INTRA_ISP) return nullptr;
  const int pw = t.comp ? W >> 1 : W, ph = t.comp ? H >> 1 : H, unit = t.comp ? 2 : 4, m = t.multiRefIdx;
  if (t.mode > B200_INTRA_MDLM_T || m > 2 || (m && t.comp)) return "bad mode / reference line";
  if (t.ciip && (t.ciip > 3 || t.mode != B200_INTRA_PLANAR)) return "bad CIIP block";
  if (t.mode >= B200_INTRA_LM && !(t.comp && t.log2w <= 5 && t.log2h <= 5 && t.lmAbove <= w && t.lmLeft <= h && (!(t.flags & B200_INTRA_LM_ABOVE) || t.y >= 2) && (!(t.flags & B200_INTRA_LM_LEFT) || t.x >= 2)
                                   && t.x + (w > 2 * t.lmAbove ? w : 2 * t.lmAbove) <= pw && t.y + (h > 2 * t.lmLeft ? h : 2 * t.lmLeft) <= ph)) return "bad CCLM block";
  if (t.mode == B200_INTRA_MIP && (t.comp || m || (t.mip & 0x7f) >= ((w == 4 && h == 4) ? 16 : (w == 4 || h == 4 || (w == 8 && h == 8)) ? 8 : 6))) return "bad MIP mode";
  if (!(t.numAbove <= 2 * w / unit && t.numLeft <= 2 * h / unit && (!t.numAbove || t.y > m) && (!t.numLeft || t.x > m)
        && (!(t.flags & B200_INTRA_AVAIL_TL) || (t.x > m && t.y > m)) && t.x + (int)t.numAbove * unit <= pw && t.y + (int)t.numLeft * unit <= ph)) return "availability outside the picture";
  return nullptr;
}

// ---- K4 / K5: per-CTU records and picture-level tables ----
// types 0..4 or OFF, BO bands 0..31, for the first nComp components
__host__ __device__ inline const char* sao_ctu_problem(const b200_sao_ctu& s, int nComp)
{
  for (int c = 0; c < nComp; c++) {
    if (s.type[c] != B200_SAO_OFF && s.type[c] > B200_SAO_BO) return "SAO type";
    if (s.type[c] == B200_SAO_BO && s.band[c] > 31) return "SAO band";
  }
  return nullptr;
}
// at most 3 boundaries per direction, on the 8x8 grid strictly inside the picture (VVC's virtual boundaries meet this by construction)
inline const char* vb_problem(const b200_vb& vb, int W, int H)
{
  if (vb.numVer < 0 || vb.numVer > 3 || vb.numHor < 0 || vb.numHor > 3) return "virtual boundaries: 0..3 per direction";
  for (int k = 0; k < vb.numVer; k++) if (vb.posX[k] <= 0 || vb.posX[k] >= W || (vb.posX[k] & 7)) return "vertical virtual boundary off the 8-sample grid or outside the picture";
  for (int k = 0; k < vb.numHor; k++) if (vb.posY[k] <= 0 || vb.posY[k] >= H || (vb.posY[k] & 7)) return "horizontal virtual boundary off the 8-sample grid or outside the picture";
  return nullptr;
}
// the 16 fixed luma sets and up to maxLumaSets - 16 APS sets: one slice has at most 8, the tables of a picture with several slices hold every slice's
// APS filters (so the other counts only have a lower bound), and a CTU record addresses 255 sets at most
inline const char* alf_tables_problem(const b200_alf_tables& T, int maxLumaSets)
{
  if (T.numLumaSets < 16 || T.numLumaSets > maxLumaSets) return maxLumaSets == 24 ? "ALF tables: numLumaSets (16..24)" : "ALF tables: numLumaSets (16..255)";
  if (T.numChromaAlts < 0 || T.numCc[0] < 0 || T.numCc[1] < 0) return "ALF tables: a negative numChromaAlts / numCc";
  return nullptr;
}
struct CtuLimits { int numLumaSets, numChromaAlts, numCc[2], numLfSlices, ctusW, ctusH; };
// every index inside its table, no undefined enable bit, and the padding forms the reference can produce (a corner is padded only where both adjacent
// sides are readable and the diagonal CTU exists; the wide chroma form only without CC-ALF on that component).  i = the CTU's raster index.
__host__ __device__ inline const char* alf_ctu_problem(const b200_alf_ctu& a, int i, const CtuLimits& lim)
{
  const int f = a.enable[0], cx = i % lim.ctusW, cy = i / lim.ctusW;
  if ((f & ~0x7f) || (a.enable[1] & ~3) || (a.enable[2] & ~3)) return "undefined ALF enable bits";
  if ((f & 1) && a.lumaSet >= lim.numLumaSets) return "lumaSet past numLumaSets";
  for (int c = 0; c < 2; c++) {
    if ((a.enable[1 + c] & 1) && a.chromaAlt[c] >= lim.numChromaAlts) return "chromaAlt past numChromaAlts";
    if (a.ccIdx[c] > lim.numCc[c]) return "ccIdx past numCc";
    if ((a.enable[1 + c] & B200_ALF_PAD_WIDE) && a.ccIdx[c]) return "PAD_WIDE with CC-ALF";
  }
  if ((f & B200_ALF_PAD_TL) && ((f & (B200_ALF_CLIP_TOP | B200_ALF_CLIP_LEFT)) || !cx || !cy)) return "PAD_TL with a clipped top / left side or on the first CTU row / column";
  if ((f & B200_ALF_PAD_BR) && ((f & (B200_ALF_CLIP_BOTTOM | B200_ALF_CLIP_RIGHT)) || cx == lim.ctusW - 1 || cy == lim.ctusH - 1)) return "PAD_BR with a clipped bottom / right side or on the last CTU row / column";
  return nullptr;
}
// T: the picture's ALF tables, or null (ALF off: every count 0)
inline CtuLimits ctu_limits(const b200_geom& g, const b200_alf_tables* T, int numLfSlices)
{
  CtuLimits l;
  l.numLumaSets = T ? T->numLumaSets : 0; l.numChromaAlts = T ? T->numChromaAlts : 0; l.numCc[0] = T ? T->numCc[0] : 0; l.numCc[1] = T ? T->numCc[1] : 0;
  l.numLfSlices = numLfSlices; l.ctusW = (g.width + g.ctuSize - 1) / g.ctuSize; l.ctusH = (g.height + g.ctuSize - 1) / g.ctuSize;
  return l;
}

// ---- LMCS: the model (b200_lmcs) and the per-VPDU records (b200_lmcs_vpdu) ----
// lmcs_vpdu_kernel walks reshapePivot[minBinIdx + 1 .. maxBinIdx + 1]; the pivots and input pivots are the ones constructReshaper (reference
// CommonLib/Reshape.cpp:317) builds from a legal APS: LmcsPivot[0] = 0, non-decreasing up to at most 2^bitDepth, InputPivot[i] = i * OrgCW
__host__ __device__ inline const char* lmcs_model_problem(const b200_lmcs& L, int bitDepth)
{
  const int org = (1 << bitDepth) / 16;
  if (L.orgCW != org) return "LMCS model: orgCW is not (1 << bitDepth) / 16";
  if (L.minBinIdx < 0 || L.minBinIdx > L.maxBinIdx || L.maxBinIdx > 15) return "LMCS model: bins (0 <= minBinIdx <= maxBinIdx <= 15)";
  if (L.reshapePivot[0] != 0) return "LMCS model: reshapePivot[0] is not 0";
  for (int i = 0; i < 16; i++) if (L.reshapePivot[i + 1] < L.reshapePivot[i]) return "LMCS model: reshapePivot decreases";
  if (L.reshapePivot[16] > (1 << bitDepth)) return "LMCS model: reshapePivot[16] above 2^bitDepth";
  for (int i = 0; i < 17; i++) if (L.inputPivot[i] != i * org) return "LMCS model: inputPivot[i] is not i * orgCW";
  return nullptr;
}
// record i of the raster of VPDUs (64x64, or the CTU when it is smaller): the CU that covers the VPDU's top-left sample starts at or above-left of it
// in the same CTU, and a neighbour is available only where it lies inside the picture.  lmcs_vpdu_kernel then reads column x - 1 and row y - 1 of the
// luma plane, clamped to its last row / column, and nothing else.
__host__ __device__ inline const char* lmcs_vpdu_problem(const b200_lmcs_vpdu& v, int i, const b200_geom& g)
{
  const int vs = g.ctuSize == 128 ? 64 : g.ctuSize, vW = (g.width + vs - 1) / vs, vx = (i % vW) * vs, vy = (i / vW) * vs, ctu = g.ctuSize;
  if (v.x >= g.width || v.y >= g.height) return "LMCS VPDU record: CU origin outside the picture";
  if ((v.availLeft && v.x == 0) || (v.availAbove && v.y == 0)) return "LMCS VPDU record: an available neighbour outside the picture";
  if (v.x > vx || v.y > vy || v.x / ctu != vx / ctu || v.y / ctu != vy / ctu) return "LMCS VPDU record: CU origin not at or above-left of its VPDU in the same CTU";
  return nullptr;
}

// ---- B200_PIC_DERIVE_LF: CU and TU records (b200_lf_cu, b200_lf_tu) ----
// lf_derive.cuh writes grid entries inside a CU's blocks and its TUs' blocks only, and reads the records a CU and TU index name: each CU record and its TUs
// must lie inside the planes they address and inside the CTU whose range lists the CU (ctu: raster index; the CTU is what calcFilterStrengthsCTU's early
// return at a slice with deblocking disabled applies to), slice and TU indices inside their arrays.
struct LfLimits { int W, H, chroma, ctuLog2, ctusW, numSlices; unsigned numTus; };
inline LfLimits lf_limits(const b200_geom& g, int numSlices, size_t numTus)
{
  LfLimits l; l.W = g.width; l.H = g.height; l.chroma = g.chromaFormat != 0; l.ctuLog2 = ctu_log2(g); l.ctusW = (g.width + g.ctuSize - 1) / g.ctuSize;
  l.numSlices = numSlices; l.numTus = (unsigned)(numTus > 0xffffffffu ? 0xffffffffu : numTus);
  return l;
}
// block (x, y, w, h) of channel type ch inside its plane and inside CTU ctu
__host__ __device__ inline bool lf_block_in_ctu(int x, int y, int w, int h, int ch, int ctu, const LfLimits& lim)
{
  const int cl = lim.ctuLog2 - ch, pw = ch ? lim.W >> 1 : lim.W, ph = ch ? lim.H >> 1 : lim.H;
  return w >= 1 && h >= 1 && x + w <= pw && y + h <= ph && (x >> cl) == ctu % lim.ctusW && (y >> cl) == ctu / lim.ctusW && ((x + w - 1) >> cl) == (x >> cl) && ((y + h - 1) >> cl) == (y >> cl);
}
__host__ __device__ inline const char* lf_cu_problem(const b200_lf_cu& c, const b200_lf_tu* tus, int ctu, const LfLimits& lim)
{
  if (c.chType > 1 || (c.chType && !lim.chroma) || c.treeType > 2 || (c.flags & ~0x7ff)) return "CU record: channel, tree type or flags";
  if (!lf_block_in_ctu(c.x, c.y, c.w, c.h, c.chType, ctu, lim)) return "CU record: block outside its plane or its CTU";
  if (c.slice >= lim.numSlices) return "CU record: slice index past numLfSlices";
  if (!c.numTus || (unsigned long long)c.firstTu + c.numTus > lim.numTus) return "CU record: TU records past numLfTus";
  for (unsigned k = 0; k < c.numTus; k++) {
    const b200_lf_tu& t = tus[c.firstTu + k];
    if ((t.w || t.h) && !lf_block_in_ctu(t.x, t.y, t.w, t.h, 0, ctu, lim)) return "TU record: luma block outside the picture or its CU's CTU";
    if ((t.cw || t.ch) && (!lim.chroma || !lf_block_in_ctu(t.cx, t.cy, t.cw, t.ch, 1, ctu, lim))) return "TU record: chroma block outside the picture or its CU's CTU";
  }
  return nullptr;
}

// ---- K3: the reach of each side of one luma edge ----
// len is the signalled length (1, 2, 3, 5 or 7).  At a CTU row (ctuRowP: a horizontal edge on a CTU's top row) the P side is never large, and beside a
// large side a short one filters as 3.  A side writes at most `writes` samples and reads `reads`: writes + 1, and 3 for lengths 1 and 2, whose decisions
// still read p2 / q2.  lf_kernel loads exactly these samples; lf_grid_problem spaces the edges of a line by them.
struct LfSide { int len, writes, reads; bool large; };
struct LfSides { LfSide p, q; };
__host__ __device__ inline LfSides lf_sides(int sideMaxFiltLength, bool ctuRowP)
{
  const int lenP = (sideMaxFiltLength >> 4) & 7, lenQ = sideMaxFiltLength & 7, nP = ctuRowP && lenP > 3 ? 3 : lenP;
  const bool large = nP > 3 || lenQ > 3;
  const auto side = [large](int len, int n) { const int w = large && n < 3 ? 3 : n; return LfSide{len, w, w < 3 ? 3 : w + 1, n > 3}; };
  return {side(lenP, nP), side(lenQ, lenQ)};
}

// ---- K3: the deblocking grid of one direction (dir 0: lfV, 1: lfH) ----
// K3's flat pass (k3_deblock.cu) is exact only when no edge reads a sample that another edge of the same direction writes, and it reads no sample outside
// the plane.  One raster scan (host only; the picture path runs the grids the glue flattens from the reference's own edge derivation unchecked); on a
// failure, (*x, *y) is the luma position of the first edge that breaks a rule.
inline const char* lf_grid_problem(const b200_geom& g, const b200_lf_param* grid, int dir, int* x, int* y)
{
  const int W4 = g.width >> 2, H4 = g.height >> 2, extent = dir ? g.height : g.width;
  const auto legal = [](int n) { return n == 1 || n == 2 || n == 3 || n == 5 || n == 7; };
  std::vector<int> prev(dir ? W4 : H4, -1), prevWQ(prev.size()), prevRQ(prev.size());   // per line: the last luma edge and its Q side's writes / reads
  for (int y4 = 0; y4 < H4; y4++)
    for (int x4 = 0; x4 < W4; x4++) {
      const b200_lf_param& e = grid[(size_t)y4 * W4 + x4];
      const int bs = e.bs & 0x3f, line = dir ? x4 : y4, pos = 4 * (dir ? y4 : x4);
      if (!bs) continue;
      *x = 4 * x4; *y = 4 * y4;
      if ((bs & 3) == 3 || ((bs >> 2) & 3) == 3 || (bs >> 4) == 3) return "Bs 3";
      if (pos == 0) return "Bs != 0 on the picture's border";
      if (!(bs & 3)) continue;                                  // chroma only: 4:2:0 chroma edges are 8 samples apart and read 4 per side
      const LfSides s = lf_sides(e.sideMaxFiltLength, dir && (pos & (g.ctuSize - 1)) == 0);
      if (!legal(s.p.len) || !legal(s.q.len)) return "luma filter lengths (1, 2, 3, 5 or 7)";
      if (pos < s.p.reads || pos + s.q.reads > extent) return "filter lengths read outside the picture";
      if (prev[line] >= 0 && (pos - prev[line] < prevWQ[line] + s.p.reads || pos - prev[line] < prevRQ[line] + s.p.writes))
        return "reads or writes samples the previous edge of its line writes or reads";
      prev[line] = pos; prevWQ[line] = s.q.writes; prevRQ[line] = s.q.reads;
    }
  return nullptr;
}

}  // namespace b200
