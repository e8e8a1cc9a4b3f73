/* k8_intra.c — CPU restatement of regular intra prediction (planar, DC, angular incl. wide angles, MRL, PDPC, BDPCM prediction).
 * TEST INFRASTRUCTURE ONLY (see vvc_oracle.h).  Follows vvdec source/Lib/CommonLib/IntraPrediction.cpp:
 *   reference samples  xFillReferenceSamples :1072-1249 (given the three availability counts), xFilterReferenceSamples :1251-1287
 *   prediction         predIntraAng :474-517, xPredIntraPlanarCore :154-210, xGetPredValDc :412-441, xPredIntraAng :592-848,
 *                      IntraPredAngleCore :301-331, IntraPredAngleChroma :333-356, IntraPredSampleFilterCore :212-238, xPredIntraBDPCM :850-885
 * Pinned by tests/test_intra_oracle_vs_ref.py against the real IntraPrediction (scalar and SIMD). */
#include "vvc_oracle.h"
#include "../vvdec_b200/csrc/vvc_tables.h"
#include <string.h>
#include <stdlib.h>

static int ilog2(int v) { int r = 0; while (v > 1) { v >>= 1; r++; } return r; }
static int iclip(int lo, int hi, int v) { return v < lo ? lo : v > hi ? hi : v; }
static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }
/* the probe of one record (orc_intra_probe): the unclipped range [lo, hi] at a clip site; NULL on the normal path */
static void seen(int32_t* lo, int32_t* hi, int v) { if (v < *lo) *lo = v; if (v > *hi) *hi = v; }
#define PROBE(site, v) do { if (pr) seen(&pr->site##Min, &pr->site##Max, (v)); } while (0)

static const int kAng[32] = {0, 1, 2, 3, 4, 6, 8, 10, 12, 14, 16, 18, 20, 23, 26, 29, 32, 35, 39, 45, 51, 57, 64, 73, 86, 102, 128, 171, 256, 341, 512, 1024};
static const int kInvAng[32] = {0, 16384, 8192, 5461, 4096, 2731, 2048, 1638, 1365, 1170, 1024, 910, 819, 712, 630, 565,
                                512, 468, 420, 364, 321, 287, 256, 224, 191, 161, 128, 96, 64, 48, 32, 16};
static const int kIntraFilterThr[2][8] = {{24, 24, 24, 14, 2, 0, 0, 0}, {40, 40, 40, 28, 4, 0, 0, 0}};   /* m_aucIntraFilter :72 */

static int wide_angle(int w, int h, int mode)     /* getWideAngle :443 */
{
  if (mode > 1 && mode <= 66) {
    static const int shift[6] = {0, 6, 10, 12, 14, 15};
    const int d = abs(ilog2(w) - ilog2(h));
    if (w > h && mode < 2 + shift[d]) mode += 65;
    else if (h > w && mode > 66 - shift[d]) mode -= 65;
  }
  return mode;
}

/* ref: (2h + mrl + 1) rows x stride (= 2w + 1 + mrl); row 0 = top-left + above row, column 0 = left column (reference layout) */
static void fill_ref(const int16_t* plane, ptrdiff_t ps, int x0, int y0, int w, int h, int mrl, int unitW, int unitH, int availTL, int numAbove, int numLeft,
                     int bitDepth, int16_t* ref, int stride, orc_intra_trace* pr)
{
  const int predSize = 2 * w, predHSize = 2 * h;
  const int totalUnits = (predSize + unitW - 1) / unitW + (predHSize + unitH - 1) / unitH + 1;
  const int16_t* src = plane + (ptrdiff_t)y0 * ps + x0;
  const int dc = 1 << (bitDepth - 1), n = availTL + numAbove + numLeft;
  if (n == 0) {
    for (int j = 0; j <= predSize + mrl; j++) ref[j] = (int16_t)dc;
    for (int i = 1; i <= predHSize + mrl; i++) ref[i * stride] = (int16_t)dc;
    PROBE(subst, dc);
  } else if (n == totalUnits) {
    const int16_t* p = src - (1 + mrl) * ps - (1 + mrl);
    for (int j = 0; j <= predSize + mrl; j++) ref[j] = p[j];
    p = src - mrl * ps - (1 + mrl);
    for (int i = 1; i <= predHSize + mrl; i++) { ref[i * stride] = *p; p += ps; }
  } else if (numLeft > 0) {
    const int16_t* p = src - (1 + mrl);
    int16_t* d = ref + (1 + mrl) * stride;
    int t = imin(numLeft * unitH, predHSize);
    for (int i = 0; i < t; i++) d[i * stride] = p[i * ps];
    for (int i = t; i < predHSize; i++) { d[i * stride] = d[(t - 1) * stride]; PROBE(subst, d[i * stride]); }
    if (availTL) {
      p = src - (1 + mrl) * ps - (1 + mrl);
      for (int j = 0; j <= mrl; j++) ref[j] = p[j];
      for (int i = 1; i <= mrl; i++) ref[i * stride] = p[i * ps];
    } else {
      const int16_t v = src[-(1 + mrl)];
      ref[0] = v;
      for (int i = 1; i <= mrl; i++) { ref[i] = v; ref[i * stride] = v; }
      PROBE(subst, v);
    }
    d = ref + 1 + mrl;
    if (numAbove) {
      p = src - ps * (1 + mrl);
      t = imin(numAbove * unitW, predSize);
      for (int j = 0; j < t; j++) d[j] = p[j];
      for (int j = t; j < predSize; j++) { d[j] = d[t - 1]; PROBE(subst, d[j]); }
    } else for (int j = 0; j < predSize; j++) { d[j] = d[-1]; PROBE(subst, d[j]); }
  } else {
    const int16_t* p = src - ps * (1 + mrl);
    int16_t* d = ref + 1 + mrl;
    const int t = imin(numAbove * unitW, predSize);
    for (int j = 0; j < t; j++) d[j] = p[j];
    for (int j = t; j < predSize; j++) { d[j] = d[t - 1]; PROBE(subst, d[j]); }
    const int16_t v = p[0];
    ref[0] = v;
    for (int i = 1; i <= mrl; i++) { ref[i] = v; ref[i * stride] = v; }
    d = ref + (1 + mrl) * stride;
    for (int i = 0; i < predHSize; i++) d[i * stride] = v;
    PROBE(subst, v);
  }
}

static void filter_ref(const int16_t* u, int16_t* f, int w, int h)      /* :1251, multiRefIdx == 0 */
{
  const int predSize = 2 * w, predHSize = 2 * h, s = predSize + 1;
  f[predHSize * s] = u[predHSize * s];
  for (int i = predHSize - 1; i >= 1; i--) f[i * s] = (int16_t)((u[(i + 1) * s] + 2 * u[i * s] + u[(i - 1) * s] + 2) >> 2);
  f[0] = (int16_t)((u[s] + 2 * u[0] + u[1] + 2) >> 2);
  for (int j = 1; j < predSize; j++) f[j] = (int16_t)((u[j + 1] + 2 * u[j] + u[j - 1] + 2) >> 2);
  f[predSize] = u[predSize];
}

#define AT(x, y) src[(y) * stride + (x)]

static void pred_planar(const int16_t* src, int stride, int w, int h, int16_t* dst, ptrdiff_t ds)
{
  const int l2w = ilog2(w), l2h = ilog2(h);
  int left[65] = {0}, top[65] = {0}, bottom[64], right[64];
  for (int k = 0; k <= w; k++) top[k] = AT(k + 1, 0);
  for (int k = 0; k <= h; k++) left[k] = AT(0, k + 1);
  const int bl = left[h], tr = top[w];
  for (int k = 0; k < w; k++) { bottom[k] = bl - top[k]; top[k] <<= l2h; }
  for (int k = 0; k < h; k++) { right[k] = tr - left[k]; left[k] <<= l2w; }
  for (int y = 0; y < h; y++) {
    int hor = left[y];
    for (int x = 0; x < w; x++) {
      hor += right[y]; top[x] += bottom[x];
      dst[y * ds + x] = (int16_t)(((hor << l2h) + (top[x] << l2w) + (1 << (l2w + l2h))) >> (1 + l2w + l2h));
    }
  }
}

/* topLen / leftLen: m_topRefLength / m_leftRefLength (2w / 2h for a regular block; CU size + partition size with ISP); waW x waH: the size the wide-angle
 * mapping looks at (the CU with ISP); isp: always the cubic filter (:745) */
static void pred_angular_ex(const int16_t* src, int stride, int w0, int h0, int chroma, int dirMode, int mrl, int doPDPC, int pmax, int16_t* dst, ptrdiff_t ds,
                            int topLen, int leftLen, int waW, int waH, int isp, orc_intra_trace* pr)
{
  int w = w0, h = h0;
  const int predMode = wide_angle(waW, waH, dirMode), ver = predMode >= 34;
  const int angMode = ver ? predMode - 50 : -(predMode - 18), absMode = abs(angMode);
  const int invAngle = kInvAng[absMode], absAng = kAng[absMode], angle = angMode < 0 ? -absAng : absAng;
  int16_t refAbove[2 * 128 + 3 + 33 * 3], refLeft[2 * 128 + 3 + 33 * 3], *refMain, *refSide;
  if (angle < 0) {
    for (int x = 0; x <= w + 1 + mrl; x++) refAbove[x + h] = AT(x, 0);
    for (int y = 0; y <= h + 1 + mrl; y++) refLeft[y + w] = AT(0, y);
    refMain = ver ? refAbove + h : refLeft + w; refSide = ver ? refLeft + w : refAbove + h;
    const int sizeSide = ver ? h : w;
    for (int k = -sizeSide; k <= -1; k++) refMain[k] = refSide[imin((-k * invAngle + 256) >> 9, sizeSide)];
  } else {
    for (int x = 0; x <= topLen + mrl; x++) refAbove[x] = AT(x, 0);
    for (int y = 0; y <= leftLen + mrl; y++) refLeft[y] = AT(0, y);
    refMain = ver ? refAbove : refLeft; refSide = ver ? refLeft : refAbove;
    const int l2r = ilog2(w) - ilog2(h), s = imax(0, ver ? l2r : -l2r), maxIndex = (mrl << s) + 2, refLength = ver ? topLen : leftLen;
    const int16_t val = refMain[refLength + mrl];
    for (int z = 1; z <= maxIndex; z++) refMain[refLength + mrl + z] = val;
  }
  int16_t tmp[64 * 64];
  const ptrdiff_t ts = ver ? ds : 64;
  int16_t* out = ver ? dst : tmp;
  if (!ver) { const int t = w; w = h; h = t; }
  refMain += mrl; refSide += mrl;
  if (angle == 0) {
    if (doPDPC) {
      const int scale = (ilog2(w) - 2 + ilog2(h) - 2 + 2) >> 2;
      const int lev[4] = {imin(3, w), imin(6, w), imin(12, w), imin(24, w)};
      const int topLeft = AT(0, 0);
      for (int y = 0; y < h; y++) {
        const int left = refSide[y + 1];
        for (int x = 0; x < lev[scale]; x++) {
          const int wL = 32 >> imin(31, (x << 1) >> scale), v = (wL * (left - topLeft) + refMain[x + 1] * 64 + 32) >> 6;
          PROBE(pdpc, v);
          out[y * ts + x] = (int16_t)iclip(0, pmax, v);
        }
        for (int x = lev[scale]; x < w; x++) out[y * ts + x] = refMain[x + 1];
      }
    } else for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) out[y * ts + x] = refMain[x + 1];
  } else {
    if (absAng & 0x1f) {
      int deltaPos = angle * (1 + mrl);
      if (!chroma) {
        const int diff = imin(abs(predMode - 18), abs(predMode - 50)), log2Size = (ilog2(w) + ilog2(h)) >> 1;
        const int interpolationFlag = diff > kIntraFilterThr[0][log2Size];       /* filterFlag, and the angle is fractional here */
        const int cubic = isp || !interpolationFlag || mrl > 0;
        if (pr) pr->interp = cubic ? 1 : 2;
        for (int y = 0; y < h; y++, deltaPos += angle) {
          const int dI = deltaPos >> 5, dF = deltaPos & 31;
          int f[4];
          if (cubic) for (int k = 0; k < 4; k++) f[k] = kIfChroma[dF * 4 + k];    /* InterpolationFilter::getChromaFilterTable(0) */
          else { f[0] = 16 - (dF >> 1); f[1] = 32 - (dF >> 1); f[2] = 16 + (dF >> 1); f[3] = dF >> 1; }   /* g_intraGaussFilter :94 */
          for (int x = 0; x < w; x++) {
            const int16_t* p = refMain + dI + x;
            int v = (int16_t)((f[0] * p[0] + f[1] * p[1] + f[2] * p[2] + f[3] * p[3] + 32) >> 6);
            if (cubic) { PROBE(cubic, v); v = iclip(0, pmax, v); }
            out[y * ts + x] = (int16_t)v;
          }
        }
      } else {
        if (pr) pr->interp = 3;
        for (int y = 0; y < h; y++, deltaPos += angle) {
          const int dI = deltaPos >> 5, dF = deltaPos & 31;
          for (int x = 0; x < w; x++) out[y * ts + x] = (int16_t)(((32 - dF) * refMain[dI + 1 + x] + dF * refMain[dI + 2 + x] + 16) >> 5);
        }
      }
    } else {
      int deltaPos = angle * (1 + mrl);
      for (int y = 0; y < h; y++, deltaPos += angle) for (int x = 0; x < w; x++) out[y * ts + x] = refMain[(deltaPos >> 5) + 1 + x];
    }
    if (angle > 0 && doPDPC) {
      const int sideSize = h;                                     /* predMode >= DIA ? block height : block width = h after the swap */
      const int angularScale = imin(2, ilog2(sideSize) - (ilog2(3 * invAngle - 2) - 8));
      if (angularScale >= 0)
        for (int y = 0; y < h; y++) {
          int invAngleSum = 256;
          for (int x = 0; x < imin(3 << angularScale, w); x++) {
            invAngleSum += invAngle;
            const int wL = 32 >> (2 * x >> angularScale), left = refSide[y + (invAngleSum >> 9) + 1], p = out[y * ts + x];
            out[y * ts + x] = (int16_t)(p + ((wL * (left - p) + 32) >> 6));
          }
        }
    }
  }
  if (!ver) for (int y = 0; y < h0; y++) for (int x = 0; x < w0; x++) dst[y * ds + x] = tmp[x * 64 + y];
}

/* Matrix intra prediction.  Follows MatrixIntraPrediction.cpp: deriveBoundaryData :67-121 (Haar down-sampling of the two boundaries, rebase on the
 * first entry), computeReducedPred :281-330 (matrix stage, transposed variant), predictionUpsampling :233-262 / predictionUpsampling1D :190-230
 * (linear interpolation, horizontally on the rows of the reduced prediction, then vertically), initPredBlockParams :139-160; size classes
 * getMipSizeId (UnitTools.cpp:3748); weights MipData.h (shift 6, offset 32). */
static void pred_mip(const int16_t* src, int stride, int w, int h, int modeIdx, int transpose, int bitDepth, int16_t* dst, ptrdiff_t ds, orc_intra_trace* pr)
{
  const int sizeId = (w == 4 && h == 4) ? 0 : (w == 4 || h == 4 || (w == 8 && h == 8)) ? 1 : 2;
  const int bdry = sizeId == 0 ? 2 : 4, red = sizeId < 2 ? 4 : 8, upH = w / red, upV = h / red, inSize = 2 * bdry;
  int top[64], left[64], in[8], inT[8];
  for (int x = 0; x < w; x++) top[x] = AT(x + 1, 0);
  for (int y = 0; y < h; y++) left[y] = AT(0, y + 1);
  for (int k = 0; k < 2; k++) {                                  /* boundaryDownsampling1D */
    const int* full = k ? left : top; const int len = k ? h : w;
    for (int d = 0; d < bdry; d++) {
      if (bdry < len) { const int f = len / bdry; int sum = 0; for (int j = 0; j < f; j++) sum += full[d * f + j]; in[k * bdry + d] = (sum + (f >> 1)) >> ilog2(f); }
      else in[k * bdry + d] = full[d];
    }
  }
  for (int d = 0; d < bdry; d++) { inT[d] = in[bdry + d]; inT[bdry + d] = in[d]; }
  int* input = transpose ? inT : in;
  const int inputOffset = input[0];
  input[0] = sizeId < 2 ? (1 << (bitDepth - 1)) - inputOffset : 0;
  if (pr) { pr->mipSizeId = sizeId; pr->mipInputOffset = inputOffset; pr->mipInput0 = input[0]; }
  for (int i = 1; i < inSize; i++) input[i] -= inputOffset;
  const uint8_t* weight = sizeId == 0 ? &kMip4x4[modeIdx * 64] : sizeId == 1 ? &kMip8x8[modeIdx * 128] : &kMip16x16[modeIdx * 448];
  const int redSize = sizeId == 2;
  int sum = 0; for (int i = 0; i < inSize; i++) sum += input[i];
  const int offset = 32 - 32 * sum, pmax = (1 << bitDepth) - 1;
  int R[64];
  for (int pos = 0; pos < red * red; pos++) {
    int acc = offset;
    for (int i = redSize; i < inSize; i++) acc += input[i] * weight[i - redSize];
    weight += inSize - redSize;
    PROBE(mip, (acc >> 6) + inputOffset);
    const int v = iclip(0, pmax, (acc >> 6) + inputOffset);
    if (transpose) R[(pos % red) * red + pos / red] = v; else R[pos] = v;
  }
  const int l2H = ilog2(upH), l2V = ilog2(upV);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      const int k = y / upV, i = y % upV;
      int hv[2];                                                  /* horizontally up-sampled value on reduced rows k - 1 and k at column x */
      for (int q = 0; q < 2; q++) {
        const int kk = k - 1 + q;
        if (kk < 0) { hv[q] = top[x]; continue; }
        if (upH == 1) { hv[q] = R[kk * red + x]; continue; }
        const int j = x / upH, ii = x % upH;
        const int before = j == 0 ? left[(kk + 1) * upV - 1] : R[kk * red + j - 1], behind = R[kk * red + j];
        hv[q] = (int16_t)((int16_t)(before * upH + (upH >> 1)) + (ii + 1) * (int16_t)(behind - before)) >> l2H;
      }
      /* the reference accumulates in Pel and shifts the wrapped sum (predictionUpsampling1D :219-224): at 12 bit x 16 the sum leaves int16 */
      dst[y * ds + x] = upV == 1 ? (int16_t)hv[1] : (int16_t)((int16_t)((int16_t)(hv[0] * upV + (upV >> 1)) + (i + 1) * (int16_t)(hv[1] - hv[0])) >> l2V);
    }
}

/* Cross-component linear model (CCLM), 4:2:0.  Follows IntraPrediction.cpp: xGetLumaRecPixels :1403-1683 (down-sampled reconstructed luma of the
 * block, one row above and one column left; 3-tap at the first row of a CTU, 5-tap for collocated chroma, else 6-tap, with edge replication where
 * the CU has no left / above neighbour), xGetLMParameters :1694-1904 (up to four template positions, min / max pairs, a = diffC * DivSig >> y,
 * b, shift), predIntraChromaLM :519-539 (clip(((a * luma) >> shift) + b), Buffer.cpp:99 linTfCore).
 * T / L: the block's unfiltered chroma reference arrays (curChroma0 = getPredictorPtr).  luma: reconstructed luma plane. */
enum { CCLM_TS = 2 * 64 + 1 };
/* the down-sampled luma (block and templates) into d0 (row -1 / column -1 hold the templates, row pitch CCLM_TS) and the parameters into p */
static void cclm_derive(const b200_geom* g, const int16_t* luma, ptrdiff_t ls, const int16_t* src, int stride, const b200_intra_tu* t, int16_t* d0, orc_cclm* p)
{
  const int w = 1 << t->log2w, h = 1 << t->log2h, mode = t->mode, unit = 2;
  const int aboveCu = (t->flags & B200_INTRA_LM_ABOVE) != 0, leftCu = (t->flags & B200_INTRA_LM_LEFT) != 0, colloc = (t->flags & B200_INTRA_LM_COLLOCATED) != 0;
  const int lx = t->x * 2, ly = t->y * 2;
  const int firstRowOfCtu = (ly & (g->ctuSize - 1)) == 0;
  const int16_t* rec = luma + (ptrdiff_t)ly * ls + lx;
  enum { TS = CCLM_TS };
  /* above template row */
  if (aboveCu) {
    /* the reference fills 2W samples for MDLM_T whatever exists there; only the lmAbove available units are ever read (:1770), so only those are made */
    const int n = mode == B200_INTRA_MDLM_T ? unit * t->lmAbove : w;
    for (int i = 0; i < n; i++) {
      const int edge = i == 0 && !leftCu;
      if (firstRowOfCtu) { const int16_t* p = rec - ls; d0[-TS + i] = (int16_t)((p[2 * i] * 2 + p[2 * i - (edge ? 0 : 1)] + p[2 * i + 1] + 2) >> 2); }
      else if (colloc) { const int16_t* p = rec - 2 * ls; d0[-TS + i] = (int16_t)((p[2 * i - ls] + p[2 * i] * 4 + p[2 * i - (edge ? 0 : 1)] + p[2 * i + 1] + p[2 * i + ls] + 4) >> 3); }
      else { const int16_t* p = rec - 2 * ls; const int m = edge ? 0 : 1;
             d0[-TS + i] = (int16_t)((p[2 * i] * 2 + p[2 * i - m] + p[2 * i + 1] + p[2 * i + ls] * 2 + p[2 * i - m + ls] + p[2 * i + 1 + ls] + 4) >> 3); }
    }
  }
  /* left template column */
  if (leftCu) {
    const int n = mode == B200_INTRA_MDLM_L ? unit * t->lmLeft : h;
    const int16_t* p = rec - 3;
    for (int j = 0; j < n; j++, p += 2 * ls) {
      if (colloc) d0[j * TS - 1] = (int16_t)((p[1 - ((j == 0 && !aboveCu) ? 0 : ls)] + p[1] * 4 + p[0] + p[2] + p[1 + ls] + 4) >> 3);
      else d0[j * TS - 1] = (int16_t)((p[1] * 2 + p[0] + p[2] + p[1 + ls] * 2 + p[ls] + p[2 + ls] + 4) >> 3);
    }
  }
  /* the block */
  for (int j = 0; j < h; j++) {
    const int16_t* p = rec + (ptrdiff_t)2 * j * ls;
    for (int i = 0; i < w; i++) {
      const int m = (i == 0 && !leftCu) ? 0 : 1;
      if (colloc) { const int up = (j == 0 && !aboveCu) ? 0 : ls; d0[j * TS + i] = (int16_t)((p[2 * i - up] + p[2 * i] * 4 + p[2 * i - m] + p[2 * i + 1] + p[2 * i + ls] + 4) >> 3); }
      else d0[j * TS + i] = (int16_t)((p[2 * i] * 2 + p[2 * i + 1] + p[2 * i - m] + p[2 * i + ls] * 2 + p[2 * i + 1 + ls] + p[2 * i - m + ls] + 4) >> 3);
    }
  }
  /* parameters */
  const int tuWU = w / unit, tuHU = h / unit;
  int aboveAvail = 0, leftAvail = 0, topNum = 0, leftNum = 0;
  if (mode == B200_INTRA_MDLM_T) { aboveAvail = t->lmAbove >= tuWU; topNum = unit * t->lmAbove; }
  else if (mode == B200_INTRA_MDLM_L) { leftAvail = t->lmLeft >= tuHU; leftNum = unit * t->lmLeft; }
  else { aboveAvail = aboveCu; leftAvail = leftCu; topNum = w; leftNum = h; }
  const int aboveIs4 = leftAvail ? 0 : 1, leftIs4 = aboveAvail ? 0 : 1;
  const int start0 = topNum >> (2 + aboveIs4), step0 = imax(1, topNum >> (1 + aboveIs4)), start1 = leftNum >> (2 + leftIs4), step1 = imax(1, leftNum >> (1 + leftIs4));
  int sl[4] = {0, 0, 0, 0}, sc[4] = {0, 0, 0, 0}, cntT = 0, cntL = 0;
  if (aboveAvail) { cntT = imin(topNum, (1 + aboveIs4) << 1); for (int k = 0, pos = start0; k < cntT; k++, pos += step0) { sl[k] = d0[-TS + pos]; sc[k] = AT(1 + pos, 0); } }
  if (leftAvail) { cntL = imin(leftNum, (1 + leftIs4) << 1); for (int k = 0, pos = start1; k < cntL; k++, pos += step1) { sl[k + cntT] = d0[pos * TS - 1]; sc[k + cntT] = AT(0, 1 + pos); } }
  if (cntT + cntL == 2) { sl[3] = sl[0]; sc[3] = sc[0]; sl[2] = sl[1]; sc[2] = sc[1]; sl[0] = sl[1]; sc[0] = sc[1]; sl[1] = sl[3]; sc[1] = sc[3]; }
  int mn[2] = {0, 2}, mx[2] = {1, 3}, *pmn = mn, *pmx = mx, tt;
  if (sl[pmn[0]] > sl[pmn[1]]) { tt = pmn[0]; pmn[0] = pmn[1]; pmn[1] = tt; }
  if (sl[pmx[0]] > sl[pmx[1]]) { tt = pmx[0]; pmx[0] = pmx[1]; pmx[1] = tt; }
  if (sl[pmn[0]] > sl[pmx[1]]) { int* q = pmn; pmn = pmx; pmx = q; }
  if (sl[pmn[1]] > sl[pmx[0]]) { tt = pmn[1]; pmn[1] = pmx[0]; pmx[0] = tt; }
  const int minL = (sl[pmn[0]] + sl[pmn[1]] + 1) >> 1, minC = (sc[pmn[0]] + sc[pmn[1]] + 1) >> 1, maxL = (sl[pmx[0]] + sl[pmx[1]] + 1) >> 1, maxC = (sc[pmx[0]] + sc[pmx[1]] + 1) >> 1;
  int a, b, shift, normDiff = -1, clamped = 0;
  if (leftAvail || aboveAvail) {
    const int diff = maxL - minL;
    if (diff > 0) {
      static const uint8_t divSig[16] = {0, 7, 6, 5, 5, 4, 4, 3, 3, 2, 2, 1, 1, 1, 1, 0};
      const int diffC = maxC - minC;
      int x = ilog2(diff);
      normDiff = (diff << 4 >> x) & 15;
      const int v = divSig[normDiff] | 8;
      x += normDiff != 0;
      const int y = diffC == 0 ? 0 : ilog2(abs(diffC)) + 1, add = 1 << y >> 1;
      a = (diffC * v + add) >> y; shift = 3 + x - y;
      if (shift < 1) { shift = 1; a = a == 0 ? 0 : a < 0 ? -15 : 15; clamped = 1; }
      b = minC - ((a * minL) >> shift);
    } else { a = 0; b = minC; shift = 0; }
  } else { a = 0; b = 1 << (g->bitDepth - 1); shift = 0; }
  p->a = a; p->b = b; p->shift = shift; p->minL = minL; p->maxL = maxL; p->minC = minC; p->maxC = maxC; p->cntT = cntT; p->cntL = cntL;
  p->normDiff = normDiff; p->clamped = clamped;
  for (int k = 0; k < 4; k++) { p->selL[k] = sl[k]; p->selC[k] = sc[k]; }
  p->blkMin = 1 << 30; p->blkMax = -1;
  for (int j = 0; j < h; j++) for (int i = 0; i < w; i++) { p->blkMin = imin(p->blkMin, d0[j * TS + i]); p->blkMax = imax(p->blkMax, d0[j * TS + i]); }
}

static void pred_cclm(const b200_geom* g, const int16_t* luma, ptrdiff_t ls, const int16_t* src, int stride, const b200_intra_tu* t, int16_t* dst, ptrdiff_t ds)
{
  static _Thread_local int16_t tmp[(64 + 1) * CCLM_TS + CCLM_TS];
  int16_t* d0 = tmp + CCLM_TS + 1;                                  /* (0,0) of the block */
  orc_cclm p;
  cclm_derive(g, luma, ls, src, stride, t, d0, &p);
  const int w = 1 << t->log2w, h = 1 << t->log2h, pmax = (1 << g->bitDepth) - 1;
  for (int j = 0; j < h; j++) for (int i = 0; i < w; i++) dst[j * ds + i] = (int16_t)iclip(0, pmax, ((p.a * d0[j * CCLM_TS + i]) >> p.shift) + p.b);
}

static void pred_angular(const int16_t* src, int stride, int w0, int h0, int chroma, int dirMode, int mrl, int filtered, int doPDPC, int pmax, int16_t* dst, ptrdiff_t ds,
                         orc_intra_trace* pr)
{
  (void)filtered;
  pred_angular_ex(src, stride, w0, h0, chroma, dirMode, mrl, doPDPC, pmax, dst, ds, 2 * w0, 2 * h0, w0, h0, 0, pr);
}

/* Intra sub-partitions (ISP), luma of one CU.  Follows IntraPrediction::initIntraPatternChTypeISP :966-1070 (the CU's reference samples are fetched
 * once; every later partition takes a window of that buffer and refreshes the row above / column left of it from the partition reconstructed just
 * before), predIntraAng / xPredIntraAng with useISP (:474, :592: wide-angle mapping by the CU size, cubic filter, PDPC only for partitions >= 4x4),
 * the 4-wide prediction regions of vertical splits of 4xN / 8xN CUs (CU::isPredRegDiffFromTB, UnitTools.cpp:3404; DecCu.cpp:341-371), partition sizes
 * CU::getISPSplitDim (UnitTools.cpp:360).  ispMode 1: horizontal split (rows), 2: vertical.  resiMask bit k: partition k adds resi (DecCu.cpp:390).
 * Test infrastructure for the next K6 slice: no device path uses this yet. */
void orc_intra_isp_cu(const b200_geom* g, int16_t* luma, const int16_t* resi, int x0, int y0, int w, int h, int ispMode, int dirMode,
                      int availTL, int numAbove, int numLeft, int leftAvail, int aboveAvail, unsigned resiMask)
{
  const ptrdiff_t ps = g->stride[0];
  const int pmax = (1 << g->bitDepth) - 1, S = 2 * w + 1, rows = 2 * h + 1;
  int16_t* B = (int16_t*)calloc((size_t)S * rows + 64, sizeof(int16_t));
  fill_ref(luma, ps, x0, y0, w, h, 0, 4, 4, availTL, numAbove, numLeft, g->bitDepth, B, S, NULL);
  const int hor = ispMode == 1, split = hor ? h : w, nonSplit = hor ? w : h;
  const int part = imax(split >> 2, nonSplit < 16 ? 16 / nonSplit : 1), nParts = split / part;
  const int regDiff = !hor && (w == 4 || (w == 8 && h > 4));                       /* vertical split with partitions narrower than 4: predict 4 wide */
  for (int k = 0; k < nParts; k++) {
    const int ox = hor ? 0 : k * part, oy = hor ? k * part : 0, tw = hor ? w : part, th = hor ? part : h;
    if (!regDiff || (ox % 4) == 0) {
      const int rw = regDiff ? 4 : tw, rh = th;
      int16_t* W = B + oy * S + ox;
      const int topLen = w + rw, leftLen = h + rh;
      const int16_t* rec = luma + (ptrdiff_t)(y0 + oy) * ps + x0 + ox;
      if (ox || oy) {
        if (hor) {
          for (int i = 0; i < rw; i++) W[1 + i] = rec[-ps + i];
          for (int i = rw; i < topLen; i++) W[1 + i] = rec[-ps + rw - 1];
          if (!leftAvail) for (int j = 0; j <= leftLen; j++) W[j * S] = rec[-ps];
        } else {
          for (int j = 0; j < rh; j++) W[(1 + j) * S] = rec[j * ps - 1];
          for (int j = rh; j < leftLen; j++) W[(1 + j) * S] = rec[(rh - 1) * ps - 1];
          if (!aboveAvail) for (int i = 0; i <= topLen; i++) W[i] = rec[-1];
        }
      }
      int16_t* dst = luma + (ptrdiff_t)(y0 + oy) * ps + x0 + ox;
      const int16_t* src = W; const int stride = S;
      const int doPDPC = rw >= 4 && rh >= 4;
      if (dirMode == 0) pred_planar(src, stride, rw, rh, dst, ps);
      else if (dirMode == 1) {
        int sum = 0; const int denom = rw == rh ? rw << 1 : imax(rw, rh);
        if (rw >= rh) for (int i = 0; i < rw; i++) sum += AT(1 + i, 0);
        if (rw <= rh) for (int i = 0; i < rh; i++) sum += AT(0, 1 + i);
        const int16_t dc = (int16_t)((sum + (denom >> 1)) >> ilog2(denom));
        for (int y = 0; y < rh; y++) for (int x = 0; x < rw; x++) dst[y * ps + x] = dc;
      } else pred_angular_ex(src, stride, rw, rh, 0, dirMode, 0, doPDPC, pmax, dst, ps, topLen, leftLen, w, h, 1, NULL);
      if (doPDPC && dirMode <= 1) {
        const int scale = (ilog2(rw) - 2 + ilog2(rh) - 2 + 2) >> 2;
        for (int y = 0; y < rh; y++) {
          const int wT = 32 >> imin(31, (y << 1) >> scale), left = AT(0, y + 1);
          for (int x = 0; x < rw; x++) { const int wL = 32 >> imin(31, (x << 1) >> scale), top = AT(x + 1, 0), v = dst[y * ps + x]; dst[y * ps + x] = (int16_t)(v + ((wL * (left - v) + wT * (top - v) + 32) >> 6)); }
        }
      }
    }
    if (resi && (resiMask >> k) & 1)
      for (int y = 0; y < th; y++) for (int x = 0; x < tw; x++) {
        const ptrdiff_t o = (ptrdiff_t)(y0 + oy + y) * ps + x0 + ox + x;
        luma[o] = (int16_t)iclip(0, pmax, luma[o] + resi[o]);
      }
  }
  free(B);
}

/* One ISP prediction region from its record (B200_INTRA_ISP, include/vvdec_b200.h): the body of orc_intra_isp_cu for region k, the CU rebuilt from the record. */
static int isp_cu_of(const b200_intra_tu* t, int* x0, int* y0, int* W, int* H)
{
  const int isp = t->mip & 3, k = (t->mip >> 2) & 3, nReg = 1 << ((t->mip >> 4) & 3), rw = 1 << t->log2w, rh = 1 << t->log2h;
  if (isp == 1) { *W = rw; *H = rh * nReg; *x0 = t->x; *y0 = t->y - k * rh; } else { *W = rw * nReg; *H = rh; *x0 = t->x - k * rw; *y0 = t->y; }
  return isp;
}
static void intra_isp_region(const b200_geom* g, int16_t* luma, const b200_intra_tu* t)
{
  int x0, y0, w, h;
  const int hor = isp_cu_of(t, &x0, &y0, &w, &h) == 1, rw = 1 << t->log2w, rh = 1 << t->log2h, ox = t->x - x0, oy = t->y - y0;
  const ptrdiff_t ps = g->stride[0];
  const int pmax = (1 << g->bitDepth) - 1, S = 2 * w + 1, rows = 2 * h + 1, dirMode = t->mode;
  const int leftAvail = t->lmLeft, aboveAvail = t->lmAbove;
  int16_t* B = (int16_t*)calloc((size_t)S * rows + 64, sizeof(int16_t));
  fill_ref(luma, ps, x0, y0, w, h, 0, 4, 4, (t->flags & B200_INTRA_AVAIL_TL) ? 1 : 0, t->numAbove, t->numLeft, g->bitDepth, B, S, NULL);
  int16_t* W = B + oy * S + ox;
  const int topLen = w + rw, leftLen = h + rh;
  const int16_t* rec = luma + (ptrdiff_t)(y0 + oy) * ps + x0 + ox;
  if (ox || oy) {
    if (hor) {
      for (int i = 0; i < rw; i++) W[1 + i] = rec[-ps + i];
      for (int i = rw; i < topLen; i++) W[1 + i] = rec[-ps + rw - 1];
      if (!leftAvail) for (int j = 0; j <= leftLen; j++) W[j * S] = rec[-ps];
    } else {
      for (int j = 0; j < rh; j++) W[(1 + j) * S] = rec[j * ps - 1];
      for (int j = rh; j < leftLen; j++) W[(1 + j) * S] = rec[(rh - 1) * ps - 1];
      if (!aboveAvail) for (int i = 0; i <= topLen; i++) W[i] = rec[-1];
    }
  }
  int16_t* dst = luma + (ptrdiff_t)(y0 + oy) * ps + x0 + ox;
  const int16_t* src = W; const int stride = S;
  const int doPDPC = rw >= 4 && rh >= 4;
  if (dirMode == 0) pred_planar(src, stride, rw, rh, dst, ps);
  else if (dirMode == 1) {
    int sum = 0; const int denom = rw == rh ? rw << 1 : imax(rw, rh);
    if (rw >= rh) for (int i = 0; i < rw; i++) sum += AT(1 + i, 0);
    if (rw <= rh) for (int i = 0; i < rh; i++) sum += AT(0, 1 + i);
    const int16_t dc = (int16_t)((sum + (denom >> 1)) >> ilog2(denom));
    for (int y = 0; y < rh; y++) for (int x = 0; x < rw; x++) dst[y * ps + x] = dc;
  } else pred_angular_ex(src, stride, rw, rh, 0, dirMode, 0, doPDPC, pmax, dst, ps, topLen, leftLen, w, h, 1, NULL);
  if (doPDPC && dirMode <= 1) {
    const int scale = (ilog2(rw) - 2 + ilog2(rh) - 2 + 2) >> 2;
    for (int y = 0; y < rh; y++) {
      const int wT = 32 >> imin(31, (y << 1) >> scale), left = AT(0, y + 1);
      for (int x = 0; x < rw; x++) { const int wL = 32 >> imin(31, (x << 1) >> scale), top = AT(x + 1, 0), v = dst[y * ps + x]; dst[y * ps + x] = (int16_t)(v + ((wL * (left - v) + wT * (top - v) + 32) >> 6)); }
    }
  }
  free(B);
}
/* width of the transform units inside an ISP region (several only where the region is wider than the sub-partitions) */
int orc_isp_tu_width(const b200_intra_tu* t)
{
  int x0, y0, w, h;
  const int isp = isp_cu_of(t, &x0, &y0, &w, &h);
  if (isp == 2 && (w == 4 || (w == 8 && h > 4))) return imax(w >> 2, h < 16 ? 16 / h : 1);
  return 1 << t->log2w;
}

/* the parameters pred_cclm derives for a CCLM record (t->mode 70..72) over the planes as they are, without predicting */
void orc_cclm_params(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* t, orc_cclm* out)
{
  const int w = 1 << t->log2w, h = 1 << t->log2h, stride = 2 * w + 1, rows = 2 * h + 1;
  int16_t* ref = (int16_t*)calloc((size_t)stride * rows + 64, sizeof(int16_t));
  static _Thread_local int16_t tmp[(64 + 1) * CCLM_TS + CCLM_TS];
  fill_ref(planes[t->comp], g->stride[t->comp], t->x, t->y, w, h, 0, 2, 2, (t->flags & B200_INTRA_AVAIL_TL) ? 1 : 0, t->numAbove, t->numLeft, g->bitDepth, ref, stride, NULL);
  cclm_derive(g, planes[0], g->stride[0], ref, stride, t, tmp + CCLM_TS + 1, out);
  free(ref);
}

static void intra_tu(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* t, orc_intra_trace* pr)
{
  if (t->flags & B200_INTRA_ISP) { intra_isp_region(g, planes[0], t); return; }
  const int c = t->comp, w = 1 << t->log2w, h = 1 << t->log2h, mrl = c ? 0 : t->multiRefIdx, pmax = (1 << g->bitDepth) - 1;
  const int unit = c ? 2 : 4, stride = 2 * w + 1 + mrl, rows = 2 * h + 1 + mrl;
  int16_t* ref = (int16_t*)calloc((size_t)stride * rows * 2 + 64, sizeof(int16_t));
  int16_t* flt = ref + (size_t)stride * rows + 32;
  fill_ref(planes[c], g->stride[c], t->x, t->y, w, h, mrl, unit, unit, (t->flags & B200_INTRA_AVAIL_TL) ? 1 : 0, t->numAbove, t->numLeft, g->bitDepth, ref, stride, pr);
  const int16_t* src = ref;
  if ((t->flags & B200_INTRA_FILTER_REF) && !c && !mrl) { filter_ref(ref, flt, w, h); src = flt; if (pr) pr->filtered = 1; }
  int16_t* dst = planes[c] + (ptrdiff_t)t->y * g->stride[c] + t->x;
  const ptrdiff_t ds = g->stride[c];
  int16_t* inter = NULL;                                        /* CIIP: the block holds the inter prediction; keep it for the blend */
  if (t->ciip) { inter = (int16_t*)malloc(sizeof(int16_t) * w * h); for (int y = 0; y < h; y++) memcpy(inter + y * w, dst + y * ds, sizeof(int16_t) * w); }
  const int doPDPC = w >= 4 && h >= 4 && mrl == 0;
  if (t->mode == B200_INTRA_PLANAR) pred_planar(src, stride, w, h, dst, ds);
  else if (t->mode == B200_INTRA_DC) {
    int sum = 0;
    const int denom = w == h ? w << 1 : imax(w, h);
    if (w >= h) for (int i = 0; i < w; i++) sum += AT(mrl + 1 + i, 0);
    if (w <= h) for (int i = 0; i < h; i++) sum += AT(0, mrl + 1 + i);
    const int16_t dc = (int16_t)((sum + (denom >> 1)) >> ilog2(denom));
    for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) dst[y * ds + x] = dc;
  } else if (t->mode == B200_INTRA_BDPCM_HOR) { for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) dst[y * ds + x] = AT(0, y + 1); }
  else if (t->mode == B200_INTRA_BDPCM_VER) { for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) dst[y * ds + x] = AT(x + 1, 0); }
  else if (t->mode >= B200_INTRA_LM) pred_cclm(g, planes[0], g->stride[0], src, stride, t, dst, ds);
  else if (t->mode == B200_INTRA_MIP) pred_mip(src, stride, w, h, t->mip & 0x7f, t->mip >> 7, g->bitDepth, dst, ds, pr);
  else pred_angular(src, stride, w, h, c != 0, t->mode, mrl, 0, doPDPC, pmax, dst, ds, pr);
  if (doPDPC && t->mode <= B200_INTRA_DC) {                    /* IntraPredSampleFilterCore :212 */
    const int scale = (t->log2w - 2 + t->log2h - 2 + 2) >> 2;
    for (int y = 0; y < h; y++) {
      const int wT = 32 >> imin(31, (y << 1) >> scale), left = AT(0, y + 1);
      for (int x = 0; x < w; x++) {
        const int wL = 32 >> imin(31, (x << 1) >> scale), top = AT(x + 1, 0), v = dst[y * ds + x];
        dst[y * ds + x] = (int16_t)(v + ((wL * (left - v) + wT * (top - v) + 32) >> 6));
      }
    }
  }
  if (inter) {                                                  /* predBlendIntraCiip :925-938 */
    const int wI = t->ciip, wM = 4 - wI;
    for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) dst[y * ds + x] = (int16_t)((wM * inter[y * w + x] + wI * dst[y * ds + x] + 2) >> 2);
    free(inter);
  }
  if (pr) for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) PROBE(pred, dst[y * ds + x]);
  free(ref);
}

void orc_intra_tu(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* t) { intra_tu(g, planes, t, NULL); }

void orc_intra_predict(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* tus, size_t numTus)
{
  for (size_t i = 0; i < numTus; i++) orc_intra_tu(g, planes, &tus[i]);
}

/* prediction + reconstruction (DecCu.cpp:390-398): blocks flagged B200_INTRA_ADD_RESI become clip(pred + resi) before the next block reads them */
static void reconstruct_tu(const b200_geom* g, int16_t* const planes[3], const int16_t* const resi[3], const b200_intra_tu* t, orc_intra_trace* pr)
{
  const int pmax = (1 << g->bitDepth) - 1;
  intra_tu(g, planes, t, pr);
  if (resi && resi[t->comp] && (t->flags & B200_INTRA_ADD_RESI)) {
    const int isp = t->flags & B200_INTRA_ISP, tw = isp ? orc_isp_tu_width(t) : 1 << t->log2w;
    for (int y = 0; y < (1 << t->log2h); y++)
      for (int x = 0; x < (1 << t->log2w); x++) {
        if (isp && !((t->ciip >> (x / tw)) & 1)) continue;                 /* transform units of the region without a residual */
        const ptrdiff_t o = (ptrdiff_t)(t->y + y) * g->stride[t->comp] + t->x + x;
        PROBE(reco, planes[t->comp][o] + resi[t->comp][o]);
        planes[t->comp][o] = (int16_t)iclip(0, pmax, planes[t->comp][o] + resi[t->comp][o]);
      }
  }
}

void orc_intra_reconstruct(const b200_geom* g, int16_t* const planes[3], const int16_t* const resi[3], const b200_intra_tu* tus, size_t numTus)
{
  for (size_t i = 0; i < numTus; i++) reconstruct_tu(g, planes, resi, &tus[i], NULL);
}

/* one record as orc_intra_reconstruct runs it (the planes advance), and what its prediction went through */
void orc_intra_probe(const b200_geom* g, int16_t* const planes[3], const int16_t* const resi[3], const b200_intra_tu* t, orc_intra_trace* out)
{
  memset(out, 0, sizeof(*out));
  out->substMin = out->cubicMin = out->pdpcMin = out->mipMin = out->recoMin = out->predMin = INT32_MAX;
  out->substMax = out->cubicMax = out->pdpcMax = out->mipMax = out->recoMax = out->predMax = INT32_MIN;
  out->mipSizeId = -1;
  reconstruct_tu(g, planes, resi, t, out);
}
