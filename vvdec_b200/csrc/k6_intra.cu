// k6_intra.cu — K6: regular intra prediction (planar, DC, angular incl. wide angles, multi reference line, PDPC, BDPCM prediction) of a
// list of transform blocks in decoding order, with the residual add that makes a block's reconstruction the next block's reference.
// Replaces (reference, source/Lib/CommonLib/IntraPrediction.cpp): xFillReferenceSamples :1072 (sample copies / substitution),
// xFilterReferenceSamples :1251, predIntraAng :474, xPredIntraPlanarCore :154, xGetPredValDc :412, xPredIntraAng :592,
// IntraPredAngleCore :301, IntraPredAngleChroma :333, IntraPredSampleFilterCore :212, xPredIntraBDPCM :850 and the pred + resi clip of
// DecCu::predAndReco (DecCu.cpp:390-398).
//
// Scheduling.  Intra blocks depend on their neighbours' reconstruction, so the list is a dataflow graph.  CTAs take blocks in order from
// a ticket counter; a block waits (bounded spin on per-block `done` words) for the earlier blocks of the list that own the units its
// available reference samples lie in (`owner` maps filled by a pre-pass, one word per 4x4 luma / 2x2 chroma unit).  Tickets are handed out
// in decoding order and only to running CTAs, so the oldest unfinished block never waits on a block that has not started: no deadlock,
// whatever the residency.  Reference samples are read with ld.global.cg (L2): another SM wrote them.
// Inside a block every sample is independent once the two reference arrays are in shared memory: one thread computes several samples.
// Both kernels (intra_kernel, intra_ctu_kernel) run the same block body, intra_block; they differ in where samples are read and results written, and in how a
// block waits for another (PlaneIo, TileIo).
#include "common.cuh"
#include <stdlib.h>
#include <string.h>
#define VVC_TABLE_QUAL static __device__ const __align__(16)
#include "vvc_tables.h"

namespace b200 {

constexpr int IT_THREADS = 128;              // threads on one block: a CTA of intra_kernel, a group of intra_ctu_kernel
constexpr int IT_REF = 2 * 64 + 8;           // top / left array: 2*size + 1 + multiRefIdx entries
constexpr int IT_ORG = 72;                   // origin of the main / side arrays (room for the negative extension, <= 64)
constexpr int IT_ARR = IT_ORG + 2 * 64 + 80; // main / side arrays (M: the projected main array of negative angles; M, S: MIP's reduced prediction and input)

// one block's shared-memory scratch: reference arrays ([0] unfiltered, [1] filtered), M / S, CCLM's down-sampled luma of the block, of the row above and of
// the column left and its (a, b, shift), DC's sum; next: intra_ctu_kernel's block tickets
struct IntraScratch {
  int16_t T[2][IT_REF], L[2][IT_REF], M[IT_ARR], S[IT_ARR], Lm[32 * 32], LmTop[64], LmLeft[64]; int LmPar[4]; int next[2], sum;
#ifdef B200_K6_PHASES
  long long clk[5];                                          // thread 0's clock64 at the start of the block and at the end of its first four phases
#endif
};

// Attribution build (-DB200_K6_PHASES, tools/k6_phases.py): cycles of each phase of intra_block summed over the blocks, per kernel (intra_kernel,
// intra_ctu_kernel) and channel (luma, chroma): wait, reference fill, reference filter, prediction and store, publish, and the block count.  Thread 0 of
// the block's threads takes the stamps; a phase that ends in a barrier includes the group's slowest thread, prediction and store end at thread 0's last
// store, so publish includes the other threads' stores, the fence and the barrier.  The default build has none of this.
#ifdef B200_K6_PHASES
__device__ unsigned long long g_k6Phases[2][2][6];
#define K6_STAMP(S, i) do { if (tid == 0) (S).clk[i] = clock64(); } while (0)
__device__ __forceinline__ void k6_phases_add(int kernel, int comp, const long long* clk)
{
  const long long end = clock64();
  unsigned long long* a = g_k6Phases[kernel][comp ? 1 : 0];
  for (int i = 0; i < 4; i++) atomicAdd(a + i, (unsigned long long)(clk[i + 1] - clk[i]));
  atomicAdd(a + 4, (unsigned long long)(end - clk[4])); atomicAdd(a + 5, 1ull);
}
#else
#define K6_STAMP(S, i) do {} while (0)
#endif

__constant__ int cAng[32] = {0, 1, 2, 3, 4, 6, 8, 10, 12, 14, 16, 18, 20, 23, 26, 29, 32, 35, 39, 45, 51, 57, 64, 73, 86, 102, 128, 171, 256, 341, 512, 1024};
__constant__ int cInvAng[32] = {0, 16384, 8192, 5461, 4096, 2731, 2048, 1638, 1365, 1170, 1024, 910, 819, 712, 630, 565,
                                512, 468, 420, 364, 321, 287, 256, 224, 191, 161, 128, 96, 64, 48, 32, 16};
__constant__ int cIntraFilterThr[8] = {24, 24, 24, 14, 2, 0, 0, 0};

struct IntraParams {
  int16_t* planes[3]; const int16_t* resi[3]; int stride[3]; int W, H, bitDepth;
  const b200_intra_tu* tus; int numTus;
  int* owner[3]; int ownerStride[3];        // per unit: index of the list entry that writes it, -1: not written by this list
  int* done; int* ticket; int* err;
  const int* perm;                          // processing order (wavefront over CTUs), or null: list order
  int* ctuCnt; int* ctuFirst; int* ctuBase; int ctuLog2, ctusW, ctusH;
  int compSel;                              // 0 all blocks, 1 luma only, 2 chroma only (second launch on the same list: the luma blocks' done words are set)
};

__device__ __forceinline__ int wide_angle(int w, int h, int mode)
{
  if (mode > 1 && mode <= 66) {
    const int d = abs((31 - __clz(w)) - (31 - __clz(h)));
    const int shift = (int)((0x0F0E0C0A0600ull >> (8 * d)) & 0xff);   // {0, 6, 10, 12, 14, 15}[d], in a register rather than a local array
    if (w > h && mode < 2 + shift) mode += 65;
    else if (h > w && mode > 66 - shift) mode -= 65;
  }
  return mode;
}

__global__ void __launch_bounds__(256) intra_owner_kernel(const IntraParams P)
{
  const int i = blockIdx.x;
  const b200_intra_tu t = P.tus[i];
  const int c = t.comp, unit = c ? 2 : 4, uw = max(1, (1 << t.log2w) / unit), uh = max(1, (1 << t.log2h) / unit);
  // ISP regions can be 1 or 2 rows high: several share a unit, the last of them completes it
  for (int k = threadIdx.x; k < uw * uh; k += blockDim.x) atomicMax(&P.owner[c][(t.y / unit + k / uw) * P.ownerStride[c] + t.x / unit + k % uw], i);
}

// Processing order.  The list is in decoding order (CTU raster); handing tickets out in that order keeps only the next few CTUs of a CTU row
// in flight.  Any topological order of the dependency graph keeps the no-deadlock argument, and so does the wavefront order
// key(CTU) = x + 2 y (left, above, above-left and above-right CTUs all have smaller keys): CTUs of one anti-diagonal run side by side.
// perm = blocks sorted by key, decoding order kept inside a CTU (its blocks are contiguous in the list).
__device__ __forceinline__ int intra_ctu_of(const IntraParams& P, const b200_intra_tu& t)
{
  const int sh = t.comp ? 1 : 0;
  return (((int)t.y << sh) >> P.ctuLog2) * P.ctusW + (((int)t.x << sh) >> P.ctuLog2);
}
__global__ void __launch_bounds__(256) intra_ctu_count_kernel(const IntraParams P)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= P.numTus) return;
  const int c = intra_ctu_of(P, P.tus[i]);
  atomicAdd(&P.ctuCnt[c], 1); atomicMin(&P.ctuFirst[c], i);
}
__global__ void intra_ctu_base_kernel(const IntraParams P)
{
  int run = 0;
  for (int d = 0; d < P.ctusW + 2 * P.ctusH; d++)
    for (int y = 0; y < P.ctusH; y++) { const int x = d - 2 * y; if (x >= 0 && x < P.ctusW) { P.ctuBase[y * P.ctusW + x] = run; run += P.ctuCnt[y * P.ctusW + x]; } }
}
__global__ void __launch_bounds__(256) intra_perm_kernel(const IntraParams P, int* perm)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= P.numTus) return;
  const int c = intra_ctu_of(P, P.tus[i]), r = i - P.ctuFirst[c];
  if (r >= P.ctuCnt[c]) { atomicOr(P.err, 2); return; }       // the CTU's blocks are not contiguous in the list
  perm[P.ctuBase[c] + r] = i;
}

// ISP regions (B200_INTRA_ISP): the neighbourhood in the record is the CU's (bx, by, bw, bh rebuilt from the region and its index); region k > 0 takes the row
// above (horizontal split) / the column left (vertical split) from the region before it, padded with its last sample, and the other side from the CU's
// reference arrays at the region's offset — or, where the CU has no neighbour on that side, the sample next to the region's corner
// (initIntraPatternChTypeISP, IntraPrediction.cpp:966-1070).  topLen / sideLen: m_topRefLength / m_leftRefLength.  Other blocks: the block itself.
struct IspGeom {
  bool isp; int bx, by, bw, bh, k, split, resiMask, l2tu, topLen, sideLen;
  __device__ __forceinline__ explicit IspGeom(const b200_intra_tu& t)
  {
    const int w = 1 << t.log2w, h = 1 << t.log2h;
    isp = t.flags & B200_INTRA_ISP; bx = t.x; by = t.y; bw = w; bh = h; k = 0; split = 0; resiMask = 0xff; l2tu = 16;
    if (isp) {
      split = t.mip & 3; k = (t.mip >> 2) & 3; const int nReg = 1 << ((t.mip >> 4) & 3);
      if (split == 1) { bh = h * nReg; by = t.y - k * h; } else { bw = w * nReg; bx = t.x - k * w; }
      int tuW = w; if (split == 2 && (bw == 4 || (bw == 8 && bh > 4))) tuW = max(bw >> 2, bh < 16 ? 16 / bh : 1);      // transform units narrower than the region
      l2tu = 31 - __clz(tuW); resiMask = t.ciip;
    }
    topLen = isp ? bw + w : 2 * w; sideLen = isp ? bh + h : 2 * h;
  }
};

__device__ __forceinline__ void intra_sync(int bar) { asm volatile("bar.sync %0, %1;" :: "r"(bar), "r"(IT_THREADS) : "memory"); }

// One record of the list, reconstructed by the IT_THREADS threads tid = 0..127 that meet at named barrier `bar`: wait for the blocks it reads from, fill
// (and filter) its reference arrays, predict, blend with CIIP's inter prediction, add the residual and store.  `io` reads samples and owner words, waits for
// an earlier block and says where results go.  The caller publishes the block after a barrier.
template <class Io>
__device__ __forceinline__ void intra_block(const IntraParams& P, const b200_intra_tu& t, const int me, const int tid, const int bar, IntraScratch& S, const Io& io)
{
  const int c = t.comp, w = 1 << t.log2w, h = 1 << t.log2h, mrl = c ? 0 : t.multiRefIdx, unit = c ? 2 : 4, ush = c ? 1 : 2;
  const int x0 = t.x, y0 = t.y, pmax = (1 << P.bitDepth) - 1;
  const int availTL = (t.flags & B200_INTRA_AVAIL_TL) ? 1 : 0, numAbove = t.numAbove, numLeft = t.numLeft;
  const IspGeom g(t);
  const int bx = g.bx, by = g.by;
  K6_STAMP(S, 0);
  if (tid == 0) S.sum = 0;
  // what reads no neighbour sample comes before the wait, which it then overlaps: the reference extents, where results go, the angular parameters
  // (bx, by, bw, bh): the block the neighbourhood was analysed for — the block itself, or the CU of an ISP region
  const int topLen = g.topLen, sideLen = g.sideLen, predSize = 2 * g.bw, predHSize = 2 * g.bh;
  const int totalUnits = (predSize + unit - 1) / unit + (predHSize + unit - 1) / unit + 1, n = availTL + numAbove + numLeft;
  const int aboveLen = min(numAbove * unit, predSize), leftLen = min(numLeft * unit, predHSize);
  const int mode = t.mode;
  const bool doPDPC = w >= 4 && h >= 4 && mrl == 0;
  // results go where `io` puts them; the CIIP inter prediction and the residual are read from the same place
  int16_t* dst = io.out(x0, y0);
  const int dp = io.pitch();
  const int16_t* rs = (P.resi[c] && (t.flags & B200_INTRA_ADD_RESI)) ? io.resi(x0, y0) : nullptr;
  const int ciipW = g.isp ? 0 : t.ciip;                      // CIIP: the block holds the inter prediction; blend (predBlendIntraCiip :925-938)
  const int predMode = wide_angle(g.bw, g.bh, mode);         // angular modes; ISP: the CU decides (:610)
  const bool ver = predMode >= 34;
  const int angMode = ver ? predMode - 50 : -(predMode - 18), absMode = abs(angMode);    // < 32 for every mode
  const int invAngle = cInvAng[absMode], absAng = cAng[absMode];

  // ---- wait for the earlier blocks this one reads from
  if (g.k && tid == 0) io.wait(me - 1);                                // ISP: the region before this one is the record before it
  for (int dep = tid; dep < 96; dep += IT_THREADS) {                   // dependency slots: 0 corner, 1..32 above units, 64..95 left units
    int ux = -1, uy = -1;
    if (dep == 0) { if (availTL) { ux = bx - 1; uy = by - 1; } }
    else if (dep <= numAbove) { ux = bx + (dep - 1) * unit; uy = by - 1; }
    else if (dep - 64 >= 0 && dep - 64 < numLeft) { ux = bx - 1; uy = by + (dep - 64) * unit; }
    if (ux >= 0 && uy >= 0) { const int o = io.owner(c, ux >> ush, uy >> ush); if (o >= 0 && o < me) io.wait(o); }
  }
  if (t.mode >= B200_INTRA_LM) {
    // CCLM reads reconstructed luma: the co-located block, up to 3 rows above and 3 columns left of it, as far as the templates go
    const bool aCu = t.flags & B200_INTRA_LM_ABOVE, lCu = t.flags & B200_INTRA_LM_LEFT;
    const int nA = max(w, aCu ? (t.mode == B200_INTRA_MDLM_T ? 2 * t.lmAbove : w) : 0), nL = max(h, lCu ? (t.mode == B200_INTRA_MDLM_L ? 2 * t.lmLeft : h) : 0);
    const int ux0 = max(0, (2 * x0 - (lCu ? 4 : 0)) >> 2), ux1 = min(P.W - 1, 2 * x0 + 2 * nA - 1) >> 2;
    const int uy0 = max(0, (2 * y0 - (aCu ? 4 : 0)) >> 2), uy1 = min(P.H - 1, 2 * y0 + 2 * nL - 1) >> 2;
    const int uw = ux1 - ux0 + 1, nU = uw * (uy1 - uy0 + 1);
    for (int u = tid; u < nU; u += IT_THREADS) { const int o = io.owner(0, ux0 + u % uw, uy0 + u / uw); if (o >= 0 && o < me) io.wait(o); }
  }
  intra_sync(bar);
  K6_STAMP(S, 1);

  // ---- reference samples (xFillReferenceSamples): T[j] = row above incl. the corner, L[i] = left column, T[0] = L[0] = corner
  auto pix = [&](int x, int y) -> int { return io.pix(c, x, y); };
  auto refT = [&](int j) -> int {                              // row above (bx, by) incl. the corner: xFillReferenceSamples :1072
    if (n == 0) return 1 << (P.bitDepth - 1);
    if (n == totalUnits) return pix(bx - 1 - mrl + j, by - 1 - mrl);
    if (j <= mrl) {                                            // corner part of the row
      if (numLeft > 0) return availTL ? pix(bx - 1 - mrl + j, by - 1 - mrl) : pix(bx - 1 - mrl, by);
      return pix(bx, by - 1 - mrl);
    }
    if (numAbove) return pix(bx + min(j - 1 - mrl, aboveLen - 1), by - 1 - mrl);
    return availTL ? pix(bx - 1, by - 1 - mrl) : pix(bx - 1 - mrl, by);      // = T[mrl]; numLeft > 0 here
  };
  auto refL = [&](int i) -> int {                              // left column, i >= 1
    if (n == 0) return 1 << (P.bitDepth - 1);
    if (n == totalUnits) return pix(bx - 1 - mrl, by - 1 - mrl + i);
    if (numLeft > 0) {
      if (i <= mrl) return availTL ? pix(bx - 1 - mrl, by - 1 - mrl + i) : pix(bx - 1 - mrl, by);
      return pix(bx - 1 - mrl, by + min(i - 1 - mrl, leftLen - 1));
    }
    return pix(bx, by - 1 - mrl);
  };
  auto regT = [&](int j) -> int {
    if (!g.k) return refT(j);
    if (g.split == 1) return j == 0 ? (t.lmLeft ? refL(y0 - by) : pix(x0, y0 - 1)) : pix(x0 + min(j - 1, w - 1), y0 - 1);
    return t.lmAbove ? refT(x0 - bx + j) : pix(x0 - 1, y0);
  };
  auto regL = [&](int i) -> int {
    if (!g.k) return refL(i);
    if (g.split == 1) return t.lmLeft ? refL(y0 - by + i) : pix(x0, y0 - 1);
    return pix(x0 - 1, y0 + min(i - 1, h - 1));
  };
  int16_t *T = S.T[0], *L = S.L[0];
  // one pass over both arrays: a thread takes entry j of the row and entry j of the column (two independent fetches in flight); entry 0 of the column is the corner
  if (!g.isp && n == totalUnits) {                             // the whole neighbourhood is available (most blocks): straight copies
    const int rx = bx - 1 - mrl, ry = by - 1 - mrl;
    for (int j = tid; j <= max(topLen, sideLen) + mrl; j += IT_THREADS) {
      const bool doT = j <= topLen + mrl, doL = j <= sideLen + mrl;
      const int vt = doT ? pix(rx + j, ry) : 0, vl = doL ? pix(rx, ry + j) : 0;
      if (doT) T[j] = (int16_t)vt;
      if (doL) L[j] = (int16_t)vl;
    }
  } else {
    for (int j = tid; j <= max(topLen, sideLen) + mrl; j += IT_THREADS) {
      const bool doT = j <= topLen + mrl, doL = j >= 1 && j <= sideLen + mrl;
      const int vt = doT ? regT(j) : 0, vl = doL ? regL(j) : 0;
      if (doT) T[j] = (int16_t)vt;
      if (doL) L[j] = (int16_t)vl;
      if (j == 0) L[0] = (int16_t)vt;
    }
  }
  intra_sync(bar);
  K6_STAMP(S, 2);
  if ((t.flags & B200_INTRA_FILTER_REF) && !c && !mrl) {     // xFilterReferenceSamples
    int16_t *FT = S.T[1], *FL = S.L[1];
    for (int j = tid; j <= predSize; j += IT_THREADS)
      FT[j] = j == 0 ? (int16_t)((L[1] + 2 * T[0] + T[1] + 2) >> 2) : j == predSize ? T[j] : (int16_t)((T[j + 1] + 2 * T[j] + T[j - 1] + 2) >> 2);
    for (int i = tid + 1; i <= predHSize; i += IT_THREADS)
      FL[i] = i == predHSize ? L[i] : (int16_t)((L[i + 1] + 2 * L[i] + L[i - 1] + 2) >> 2);
    intra_sync(bar);
    if (tid == 0) FL[0] = FT[0];
    T = FT; L = FL;
    intra_sync(bar);
  }
  K6_STAMP(S, 3);

  auto store = [&](int x, int y, int v) {
    int16_t* d = dst + y * dp + x;
    if (ciipW) v = ((4 - ciipW) * (int)*d + ciipW * v + 2) >> 2;
    if (rs && ((g.resiMask >> (x >> g.l2tu)) & 1)) v = clip3(0, pmax, v + rs[y * dp + x]);
    io.put(d, x0 + x, y0 + y, v);
  };

  if (mode == B200_INTRA_PLANAR || mode == B200_INTRA_DC) {
    int dc = 0;
    if (mode == B200_INTRA_DC) {                             // xGetPredValDc
      int part = 0;
      for (int i = tid; i < w + h; i += IT_THREADS) {
        if (i < w) { if (w >= h) part += T[mrl + 1 + i]; }
        else if (w <= h) part += L[mrl + 1 + i - w];
      }
      for (int o = 16; o; o >>= 1) part += __shfl_down_sync(0xffffffffu, part, o);
      if ((tid & 31) == 0 && part) atomicAdd(&S.sum, part);
      intra_sync(bar);
      const int denom = w == h ? w << 1 : max(w, h);
      dc = (S.sum + (denom >> 1)) >> (31 - __clz(denom));
    }
    const int l2w = t.log2w, l2h = t.log2h, scale = (l2w - 2 + l2h - 2 + 2) >> 2;
    const int bl = L[h + 1], tr = T[w + 1];
#pragma unroll 2
    for (int k = tid; k < w * h; k += IT_THREADS) {
      const int y = k >> l2w, x = k & (w - 1);
      int v;
      if (mode == B200_INTRA_PLANAR) {                       // xPredIntraPlanarCore in closed form
        const int hor = (L[y + 1] << l2w) + (x + 1) * (tr - L[y + 1]), vert = (T[x + 1] << l2h) + (y + 1) * (bl - T[x + 1]);
        v = ((hor << l2h) + (vert << l2w) + (1 << (l2w + l2h))) >> (1 + l2w + l2h);
      } else v = dc;
      v = (int16_t)v;
      if (doPDPC) {                                          // IntraPredSampleFilterCore
        const int wT = 32 >> min(31, (y << 1) >> scale), wL = 32 >> min(31, (x << 1) >> scale);
        v = (int16_t)(v + ((wL * (L[y + 1] - v) + wT * (T[x + 1] - v) + 32) >> 6));
      }
      store(x, y, v);
    }
  } else if (mode >= B200_INTRA_LM) {
    // ---- cross-component linear model (xGetLumaRecPixels, xGetLMParameters, predIntraChromaLM), 4:2:0: luma at (lx0 + dx, ly0 + dy)
    const bool aCu = t.flags & B200_INTRA_LM_ABOVE, lCu = t.flags & B200_INTRA_LM_LEFT, colloc = t.flags & B200_INTRA_LM_COLLOCATED;
    const int lx0 = 2 * x0, ly0 = 2 * y0;
    const bool firstRowOfCtu = ((2 * y0) & ((1 << P.ctuLog2) - 1)) == 0;
    const int nTop = aCu ? (mode == B200_INTRA_MDLM_T ? 2 * t.lmAbove : w) : 0, nLeft = lCu ? (mode == B200_INTRA_MDLM_L ? 2 * t.lmLeft : h) : 0;
    auto ly = [&](int dx, int dy) -> int { return io.pix(0, lx0 + dx, ly0 + dy); };
    for (int k = tid; k < nTop + nLeft + w * h; k += IT_THREADS) {
      if (k < nTop) {                                          // row above the block
        const int i = k, m = (i == 0 && !lCu) ? 0 : 1;
        int v;
        if (firstRowOfCtu) v = (ly(2 * i, -1) * 2 + ly(2 * i - m, -1) + ly(2 * i + 1, -1) + 2) >> 2;
        else if (colloc) v = (ly(2 * i, -3) + ly(2 * i, -2) * 4 + ly(2 * i - m, -2) + ly(2 * i + 1, -2) + ly(2 * i, -1) + 4) >> 3;
        else v = (ly(2 * i, -2) * 2 + ly(2 * i - m, -2) + ly(2 * i + 1, -2) + ly(2 * i, -1) * 2 + ly(2 * i - m, -1) + ly(2 * i + 1, -1) + 4) >> 3;
        S.LmTop[i] = (int16_t)v;
      } else if (k < nTop + nLeft) {                           // column left of the block
        const int j = k - nTop;
        int v;
        if (colloc) v = (ly(-2, 2 * j - ((j == 0 && !aCu) ? 0 : 1)) + ly(-2, 2 * j) * 4 + ly(-3, 2 * j) + ly(-1, 2 * j) + ly(-2, 2 * j + 1) + 4) >> 3;
        else v = (ly(-2, 2 * j) * 2 + ly(-3, 2 * j) + ly(-1, 2 * j) + ly(-2, 2 * j + 1) * 2 + ly(-3, 2 * j + 1) + ly(-1, 2 * j + 1) + 4) >> 3;
        S.LmLeft[j] = (int16_t)v;
      } else {                                                 // the block
        const int q = k - nTop - nLeft, j = q >> t.log2w, i = q & (w - 1), m = (i == 0 && !lCu) ? 0 : 1;
        int v;
        if (colloc) { const int up = (j == 0 && !aCu) ? 0 : 1; v = (ly(2 * i, 2 * j - up) + ly(2 * i, 2 * j) * 4 + ly(2 * i - m, 2 * j) + ly(2 * i + 1, 2 * j) + ly(2 * i, 2 * j + 1) + 4) >> 3; }
        else v = (ly(2 * i, 2 * j) * 2 + ly(2 * i + 1, 2 * j) + ly(2 * i - m, 2 * j) + ly(2 * i, 2 * j + 1) * 2 + ly(2 * i + 1, 2 * j + 1) + ly(2 * i - m, 2 * j + 1) + 4) >> 3;
        S.Lm[q] = (int16_t)v;
      }
    }
    intra_sync(bar);
    if (tid == 0) {                                            // xGetLMParameters: four template positions -> a, b, shift
      const int tuWU = w >> 1, tuHU = h >> 1;
      bool aboveAvail = false, leftAvail = false; int topNum = 0, leftNum = 0;
      if (mode == B200_INTRA_MDLM_T) { aboveAvail = t.lmAbove >= tuWU; topNum = 2 * t.lmAbove; }
      else if (mode == B200_INTRA_MDLM_L) { leftAvail = t.lmLeft >= tuHU; leftNum = 2 * t.lmLeft; }
      else { aboveAvail = aCu; leftAvail = lCu; topNum = w; leftNum = h; }
      const int aboveIs4 = leftAvail ? 0 : 1, leftIs4 = aboveAvail ? 0 : 1;
      const int start0 = topNum >> (2 + aboveIs4), step0 = max(1, topNum >> (1 + aboveIs4)), start1 = leftNum >> (2 + leftIs4), step1 = max(1, leftNum >> (1 + leftIs4));
      int sl[4] = {0, 0, 0, 0}, sc[4] = {0, 0, 0, 0}, cntT = 0, cntL = 0;
      if (aboveAvail) { cntT = min(topNum, (1 + aboveIs4) << 1); for (int q = 0, pos = start0; q < cntT; q++, pos += step0) { sl[q] = S.LmTop[pos]; sc[q] = T[1 + pos]; } }
      if (leftAvail) { cntL = min(leftNum, (1 + leftIs4) << 1); for (int q = 0, pos = start1; q < cntL; q++, pos += step1) { sl[q + cntT] = S.LmLeft[pos]; sc[q + cntT] = L[1 + pos]; } }
      if (cntT + cntL == 2) { sl[3] = sl[0]; sc[3] = sc[0]; sl[2] = sl[1]; sc[2] = sc[1]; sl[0] = sl[1]; sc[0] = sc[1]; sl[1] = sl[3]; sc[1] = sc[3]; }
      int mn0 = 0, mn1 = 2, mx0 = 1, mx1 = 3, tt;
      if (sl[mn0] > sl[mn1]) { tt = mn0; mn0 = mn1; mn1 = tt; }
      if (sl[mx0] > sl[mx1]) { tt = mx0; mx0 = mx1; mx1 = tt; }
      if (sl[mn0] > sl[mx1]) { tt = mn0; mn0 = mx0; mx0 = tt; tt = mn1; mn1 = mx1; mx1 = tt; }     // the two groups change roles
      if (sl[mn1] > sl[mx0]) { tt = mn1; mn1 = mx0; mx0 = tt; }
      const int minL = (sl[mn0] + sl[mn1] + 1) >> 1, minC = (sc[mn0] + sc[mn1] + 1) >> 1, maxL = (sl[mx0] + sl[mx1] + 1) >> 1, maxC = (sc[mx0] + sc[mx1] + 1) >> 1;
      int a = 0, b = 1 << (P.bitDepth - 1), shift = 0;
      if (leftAvail || aboveAvail) {
        const int diff = maxL - minL;
        if (diff > 0) {
          const int diffC = maxC - minC;
          int x = 31 - __clz(diff);
          const int normDiff = (diff << 4 >> x) & 15;
          const int v = (int)((0x0765544332211110ull >> (4 * (15 - normDiff))) & 15) | 8;   // DivSigTable {0,7,6,5,5,4,4,3,3,2,2,1,1,1,1,0}
          x += normDiff != 0;
          const int y = diffC == 0 ? 0 : (31 - __clz(abs(diffC))) + 1, add = 1 << y >> 1;
          a = (diffC * v + add) >> y; shift = 3 + x - y;
          if (shift < 1) { shift = 1; a = a == 0 ? 0 : a < 0 ? -15 : 15; }
          b = minC - ((a * minL) >> shift);
        } else { a = 0; b = minC; shift = 0; }
      }
      S.LmPar[0] = a; S.LmPar[1] = b; S.LmPar[2] = shift;
    }
    intra_sync(bar);
    const int a = S.LmPar[0], b = S.LmPar[1], shift = S.LmPar[2];
    for (int k = tid; k < w * h; k += IT_THREADS) { const int y = k >> t.log2w, x = k & (w - 1); store(x, y, clip3(0, pmax, ((a * S.Lm[k]) >> shift) + b)); }
  } else if (mode == B200_INTRA_MIP) {
    // ---- matrix intra prediction (PredictorMIP): reduced boundary -> matrix stage -> linear up-sampling; M holds the reduced prediction
    const int sizeId = (w == 4 && h == 4) ? 0 : (w == 4 || h == 4 || (w == 8 && h == 8)) ? 1 : 2;
    const int bdry = sizeId == 0 ? 2 : 4, red = sizeId < 2 ? 4 : 8, upH = w / red, upV = h / red, inSize = 2 * bdry;
    const int modeIdx = t.mip & 0x7f; const bool transpose = t.mip >> 7;
    int16_t* in = S.S; int16_t* sM = S.M;                      // the (rebased) input vector, [inSize]
    if (tid < inSize) {                                        // boundaryDownsampling1D of the top / left boundary, in the order the matrix wants
      const bool fromLeft = (tid >= bdry) != transpose; const int d = tid % bdry, len = fromLeft ? h : w;
      const int16_t* full = (fromLeft ? L : T) + 1;
      int v;
      if (bdry < len) { const int f = len / bdry; int sum = 0; for (int j = 0; j < f; j++) sum += full[d * f + j]; v = (sum + (f >> 1)) >> (31 - __clz(f)); }
      else v = full[d];
      in[tid] = (int16_t)v;
    }
    intra_sync(bar);
    const int inputOffset = in[0];
    intra_sync(bar);
    if (tid < inSize) in[tid] = (int16_t)(tid == 0 ? (sizeId < 2 ? (1 << (P.bitDepth - 1)) - inputOffset : 0) : in[tid] - inputOffset);
    intra_sync(bar);
    for (int o = tid; o < red * red; o += IT_THREADS) {        // computeReducedPred: one output per thread
      const int redSize = sizeId == 2, stride = inSize - redSize;
      const uint8_t* wgt = (sizeId == 0 ? kMip4x4 + modeIdx * 64 : sizeId == 1 ? kMip8x8 + modeIdx * 128 : kMip16x16 + modeIdx * 448) + o * stride;
      int sum = 0, acc = 0;
      for (int i = 0; i < inSize; i++) sum += in[i];
      for (int i = redSize; i < inSize; i++) acc += in[i] * wgt[i - redSize];
      const int v = clip3(0, pmax, ((acc + 32 - 32 * sum) >> 6) + inputOffset);
      sM[transpose ? (o % red) * red + o / red : o] = (int16_t)v;
    }
    intra_sync(bar);
    const int l2H = 31 - __clz(upH), l2V = 31 - __clz(upV);
    for (int k = tid; k < w * h; k += IT_THREADS) {
      const int y = k >> t.log2w, x = k & (w - 1), kr = y / upV, i = y % upV;
      int hv[2];                                               // horizontally up-sampled rows kr - 1 (or the top boundary) and kr at column x
#pragma unroll
      for (int q = 0; q < 2; q++) {
        const int k2 = kr - 1 + q;
        if (k2 < 0) hv[q] = T[x + 1];
        else if (upH == 1) hv[q] = sM[k2 * red + x];
        else {
          const int j = x / upH, ii = x % upH, before = j == 0 ? L[(k2 + 1) * upV] : sM[k2 * red + j - 1], behind = sM[k2 * red + j];
          hv[q] = (int16_t)(before * upH + (upH >> 1) + (ii + 1) * (behind - before)) >> l2H;   // the reference accumulates in Pel (int16): wraps at 12 bit x 16
        }
      }
      store(x, y, upV == 1 ? hv[1] : (int16_t)(hv[0] * upV + (upV >> 1) + (i + 1) * (hv[1] - hv[0])) >> l2V);
    }
  } else if (mode >= B200_INTRA_BDPCM_HOR) {
    for (int k = tid; k < w * h; k += IT_THREADS) { const int y = k >> t.log2w, x = k & (w - 1); store(x, y, mode == B200_INTRA_BDPCM_HOR ? L[y + 1] : T[x + 1]); }
  } else {
    // ---- angular (xPredIntraAng): every sample on its own from the main / side references
    const int angle = angMode < 0 ? -absAng : absAng;
    const int16_t *mainSrc = ver ? T : L, *sideSrc = ver ? L : T;
    const int mw = ver ? w : h, mh = ver ? h : w;            // block size along the main / the side reference
    // angles >= 0 read the main reference directly, clamped to its end (the replication tail of xPredIntraAng); negative angles stage the main array
    // with the side reference projected in front of it.  Only angles >= 0 read the side reference.
    const int16_t *Mp, *Sp = sideSrc + mrl;
    int mEnd;                                                  // last main index read as is: later ones read entry mEnd
    if (angle < 0) {
      int16_t* M = S.M + IT_ORG;
      for (int k = tid - mh; k <= mw + 1 + mrl; k += IT_THREADS) M[k] = k >= 0 ? mainSrc[k] : sideSrc[min((-k * invAngle + 256) >> 9, mh)];
      intra_sync(bar);
      Mp = M + mrl; mEnd = 1 << 20;
    } else { Mp = mainSrc + mrl; mEnd = ver ? topLen : sideLen; }
    auto ref = [&](int i) -> int { return Mp[min(i, mEnd)]; };
    const int l2mw = 31 - __clz(mw), l2mh = 31 - __clz(mh);
    const int topLeft = T[0];
    const int scale0 = (l2mw - 2 + l2mh - 2 + 2) >> 2;
    const int lev = min(3 << scale0, mw);                    // lev[scale] = min(3, 6, 12, 24; width)
    const bool frac = (absAng & 31) != 0;
    const int diff = min(abs(predMode - 18), abs(predMode - 50));
    const bool cubic = g.isp || !(diff > cIntraFilterThr[(l2mw + l2mh) >> 1]) || mrl > 0;
    int angularScale = -1;
    if (angle > 0 && doPDPC) angularScale = min(2, l2mh - ((31 - __clz(3 * invAngle - 2)) - 8));
#pragma unroll 2
    for (int k = tid; k < mw * mh; k += IT_THREADS) {
      const int yy = k >> l2mw, xx = k & (mw - 1);
      int v;
      if (angle == 0) {
        if (doPDPC && xx < lev) { const int wL = 32 >> min(31, (xx << 1) >> scale0); v = clip3(0, pmax, (wL * (Sp[yy + 1] - topLeft) + ref(xx + 1) * 64 + 32) >> 6); }
        else v = ref(xx + 1);
      } else {
        const int deltaPos = angle * (1 + mrl + yy), dI = deltaPos >> 5, dF = deltaPos & 31;
        if (!frac) v = ref(dI + 1 + xx);
        else if (c) v = (int16_t)(((32 - dF) * ref(dI + 1 + xx) + dF * ref(dI + 2 + xx) + 16) >> 5);
        else {
          const int p = dI + xx;
          int f0, f1, f2, f3;
          if (cubic) { f0 = kIfChroma[dF * 4]; f1 = kIfChroma[dF * 4 + 1]; f2 = kIfChroma[dF * 4 + 2]; f3 = kIfChroma[dF * 4 + 3]; }
          else { f0 = 16 - (dF >> 1); f1 = 32 - (dF >> 1); f2 = 16 + (dF >> 1); f3 = dF >> 1; }
          v = (int16_t)((f0 * ref(p) + f1 * ref(p + 1) + f2 * ref(p + 2) + f3 * ref(p + 3) + 32) >> 6);
          if (cubic) v = clip3(0, pmax, v);
        }
        if (angularScale >= 0 && xx < min(3 << angularScale, mw)) {
          const int invAngleSum = 256 + (xx + 1) * invAngle, wL = 32 >> (2 * xx >> angularScale), left = Sp[yy + (invAngleSum >> 9) + 1];
          v = (int16_t)(v + ((wL * (left - v) + 32) >> 6));
        }
      }
      if (ver) store(xx, yy, v); else store(yy, xx, v);
    }
  }
  K6_STAMP(S, 4);
}

// intra_kernel: samples, owner words and done words in global memory; a block's results go to the plane
struct PlaneIo {
  const IntraParams& P; const int c;
  __device__ __forceinline__ int pix(int comp, int x, int y) const { return __ldcg(P.planes[comp] + (size_t)y * P.stride[comp] + x); }
  __device__ __forceinline__ int owner(int comp, int ux, int uy) const { return P.owner[comp][uy * P.ownerStride[comp] + ux]; }
  __device__ __forceinline__ void wait(int o) const
  {
    const volatile int* d = P.done + o; const volatile int* e = P.err;
    int spins = 0;
    while (*d == 0) { __nanosleep(64); if (*e || ++spins > (1 << 22)) { atomicOr(P.err, 1); break; } }   // bounded: a broken list must not hang the GPU
    __threadfence();
  }
  __device__ __forceinline__ int16_t* out(int x, int y) const { return P.planes[c] + (size_t)y * P.stride[c] + x; }
  __device__ __forceinline__ int pitch() const { return P.stride[c]; }
  __device__ __forceinline__ const int16_t* resi(int x, int y) const { return P.resi[c] + (size_t)y * P.stride[c] + x; }
  __device__ __forceinline__ void put(int16_t* d, int, int, int v) const { *d = (int16_t)v; }
};

__global__ void __launch_bounds__(IT_THREADS, 12) intra_kernel(const IntraParams P)
{
  __shared__ IntraScratch S;
  __shared__ int sTicket;
  const int tid = threadIdx.x;
  for (;;) {
    __syncthreads();
    if (tid == 0) sTicket = atomicAdd(P.ticket, 1);
    __syncthreads();
    if (sTicket >= P.numTus) return;
    if (P.perm && (*(volatile int*)P.err & 2)) return;          // the list is not in decoding order (CTU runs not contiguous): perm holds holes, nothing is run
    const int me = P.perm ? P.perm[sTicket] : sTicket;
    const b200_intra_tu t = P.tus[me];
    if ((P.compSel == 1 && t.comp != 0) || (P.compSel == 2 && t.comp == 0)) continue;      // the other channel's pass
    intra_block(P, t, me, tid, 0, S, PlaneIo{P, t.comp});
    // ---- publish
    __threadfence();
    __syncthreads();
    if (tid == 0) atomicExch(P.done + me, 1);
#ifdef B200_K6_PHASES
    if (tid == 0) k6_phases_add(0, t.comp, S.clk);
#endif
  }
}

// ================================================================================================ K6 v2: one CTA per CTU, the CTU resident in shared memory
// The dependency chains of an intra picture run block to block; v1 pays a global-memory round trip per hop (ticket, owner lookup, done flag, reference
// samples through L2: ~4 us).  v2 keeps the hops on chip: a CTA owns one CTU at a time (CTUs handed out in wave-front order, key x + 2 y), loads the
// CTU's samples (inter prediction + residual reconstruction so far) and residual planes into shared memory, and its groups take the CTU's blocks in
// decoding order — one group per block, every sample of a block independent once the reference arrays are built.  A block waits on shared-memory done
// flags for earlier blocks of its own CTU and on the global done words only for blocks of the neighbouring CTUs (left, above-left, above, above-right:
// all earlier in the wave front, so the oldest unfinished block never waits on a block that has not been started — no deadlock at any residency).
// Samples are written through: to the shared tile for the CTU's own later blocks, to the plane for the other CTUs and the in-loop filters.
// a block is worked on by a group of IT_THREADS threads, V2_GROUPS blocks of the CTU at a time (the chains of an intra CTU are Y -> Y -> Y, Cb -> Cb,
// Cr -> Cr, so about three blocks can run at once and the latency of one block is what counts)
constexpr int V2_GROUPS = 5, V2_THREADS = IT_THREADS * V2_GROUPS;
constexpr int V2_LS = 136, V2_CS = 72;                       // tile row pitch in samples: a multiple of 16 bytes (16-byte asynchronous copies), rows 4 banks apart
constexpr int V2_TILE = 128 * V2_LS + 2 * 64 * V2_CS;        // samples of one tile set (Y, Cb, Cr)
constexpr int V2_RECS = 1024;                                // records staged in shared memory (a CTU with more blocks reads the rest from global memory)
constexpr int V2_FLAGS = 128 * 128 / 16 + 2 * (64 * 64 / 4); // most blocks a CTU can hold without overlapping records (a list with more is refused)
static_assert(V2_FLAGS == INTRA_MAX_CTU_BLOCKS, "the documented per-CTU block limit is the number of done bytes");
constexpr int V2_OWN = 3 * 32 * 32;                         // owner words of the CTU's units: luma 32 x 32 (4x4 units), Cb / Cr 32 x 32 each (2x2 units)
constexpr size_t V2_SMEM = (size_t)2 * V2_TILE * sizeof(int16_t) + V2_GROUPS * sizeof(IntraScratch) + V2_RECS * sizeof(b200_intra_tu) + V2_OWN * sizeof(int) + V2_FLAGS + 64;
__device__ __forceinline__ int v2_tile_off(int c) { return c == 0 ? 0 : c == 1 ? 128 * V2_LS : 128 * V2_LS + 64 * V2_CS; }     // component c in a tile set

// CTUs that hold blocks, sorted by the wave-front key (x + 2 y, then y): every CTU counts the non-empty CTUs that precede it
__global__ void __launch_bounds__(1024) intra_ctu_order_kernel(const IntraParams P, int* ctuOrder, int* counters)
{
  extern __shared__ int sCnt[];
  const int n = P.ctusW * P.ctusH;
  for (int i = threadIdx.x; i < n; i += blockDim.x) sCnt[i] = P.ctuCnt[i];
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (sCnt[i] <= 0) continue;
    const int y = i / P.ctusW, x = i - y * P.ctusW, key = x + 2 * y;
    int rank = 0;
    for (int j = 0; j < n; j++) { const int yj = j / P.ctusW, kj = (j - yj * P.ctusW) + 2 * yj; rank += (sCnt[j] > 0) && (kj < key || (kj == key && yj < y)); }
    ctuOrder[rank] = i;
  }
  if (threadIdx.x == 0) { int m = 0; for (int j = 0; j < n; j++) m += sCnt[j] > 0; counters[0] = m; counters[1] = 0; }
}
// contiguity of every CTU's blocks in the list (decoding order): entry i belongs to the run [ctuFirst, ctuFirst + ctuCnt) of its CTU; and no CTU holds more
// blocks than intra_ctu_kernel has done bytes for (only overlapping records get there)
__global__ void __launch_bounds__(256) intra_ctu_check_kernel(const IntraParams P)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= P.numTus) return;
  const int c = intra_ctu_of(P, P.tus[i]);
  if (i - P.ctuFirst[c] >= P.ctuCnt[c]) atomicOr(P.err, INTRA_ERR_ORDER);
  if (i == P.ctuFirst[c] && P.ctuCnt[c] > V2_FLAGS) atomicOr(P.err, INTRA_ERR_CTU_BLOCKS);
}

__device__ __forceinline__ int v2_ld_acquire(const int* p) { int v; asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void v2_st_release(int* p, int v) { asm volatile("st.release.gpu.global.b32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }


// intra_ctu_kernel: the CTU's samples, residuals and owner words in shared memory (the CTU at luma (cx, cy), cw x ch samples; component c's tile is these
// >> (c ? 1 : 0), at v2_tile_off(c) in the tile sets), the planes around it; a block's results go to the tile and through to the plane.  The component is a
// plain value, not an index into arrays of tile origins: such an array would live in local memory.
struct TileIo {
  const IntraParams& P; int16_t* tile; const int* sown; const volatile uint8_t* sflag; const int first, cx, cy, cw, ch, c;
  __device__ __forceinline__ int pix(int comp, int x, int y) const
  {
    const int s = comp ? 1 : 0, tx = x - (cx >> s), ty = y - (cy >> s);
    return ((unsigned)tx < (unsigned)(cw >> s) && (unsigned)ty < (unsigned)(ch >> s)) ? (int)tile[v2_tile_off(comp) + ty * (s ? V2_CS : V2_LS) + tx]
                                                                                     : (int)__ldcg(P.planes[comp] + (size_t)y * P.stride[comp] + x);
  }
  __device__ __forceinline__ int owner(int comp, int ux, int uy) const     // inside the CTU: the staged owner word (4x4 luma and 2x2 chroma units are 4 luma samples wide)
  {
    const int ox = ux - (cx >> 2), oy = uy - (cy >> 2);
    return ((unsigned)ox < 32u && (unsigned)oy < 32u && ux * 4 < cx + cw && uy * 4 < cy + ch) ? sown[comp * 1024 + oy * 32 + ox]
                                                                                             : __ldcg(P.owner[comp] + (size_t)uy * P.ownerStride[comp] + ux);
  }
  // waits for the earlier block o with acquire semantics: the group barrier after the waits orders the group's reads of the block's samples behind it —
  // shared-memory done bytes for blocks of this CTU (CTA scope), the global done words for the others (GPU scope)
  __device__ __forceinline__ void wait(int o) const
  {
    int spins = 0;
    if (o >= first) {
      // every re-poll sleeps 20 ns: the 4K I picture's K6 is 0.8 % faster than with 64 tight spins first, and slower with 100 or 300 ns (H100, 700 W)
      while (sflag[o - first] == 0) { __nanosleep(20); if (++spins > (1 << 24)) { atomicOr(P.err, 1); break; } }
      __threadfence_block();
      return;
    }
    const volatile int* e = P.err;
    while (v2_ld_acquire(P.done + o) == 0) { __nanosleep(32); if (*e || ++spins > (1 << 22)) { atomicOr(P.err, 1); break; } }
  }
  __device__ __forceinline__ int16_t* out(int x, int y) const { const int s = c ? 1 : 0; return tile + v2_tile_off(c) + (y - (cy >> s)) * pitch() + (x - (cx >> s)); }
  __device__ __forceinline__ int pitch() const { return c ? V2_CS : V2_LS; }
  __device__ __forceinline__ const int16_t* resi(int x, int y) const { return out(x, y) + V2_TILE; }
  __device__ __forceinline__ void put(int16_t* d, int x, int y, int v) const { *d = (int16_t)v; P.planes[c][(size_t)y * P.stride[c] + x] = (int16_t)v; }
};

__global__ void __launch_bounds__(V2_THREADS, 1) intra_ctu_kernel(const IntraParams P, const int* __restrict__ ctuOrder, int* counters)
{
  extern __shared__ __align__(16) unsigned char smem[];
  int16_t* tileRec = reinterpret_cast<int16_t*>(smem);
  int16_t* tileRes = tileRec + V2_TILE;
  IntraScratch* scratch = reinterpret_cast<IntraScratch*>(tileRes + V2_TILE);
  b200_intra_tu* srec = reinterpret_cast<b200_intra_tu*>(scratch + V2_GROUPS);
  int* sown = reinterpret_cast<int*>(srec + V2_RECS);
  volatile uint8_t* sflag = reinterpret_cast<volatile uint8_t*>(sown + V2_OWN);
  __shared__ int sCtu, sNext;
  const int tid = threadIdx.x, lane = tid & (IT_THREADS - 1), grp = tid / IT_THREADS;      // lane: index inside the group
  const int nComp = P.planes[1] ? 3 : 1;
  const int ctuSize = 1 << P.ctuLog2;
  for (;;) {
    __syncthreads();
    if (tid == 0) { sCtu = atomicAdd(&counters[1], 1); sNext = V2_GROUPS; }
    __syncthreads();
    if (sCtu >= counters[0] || (*(volatile int*)P.err & (INTRA_ERR_ORDER | INTRA_ERR_CTU_BLOCKS))) return;   // intra_ctu_check_kernel: a CTU's blocks are not
                                                                             // contiguous in the list, or more than sflag holds: nothing is staged
    const int ctu = ctuOrder[sCtu], first = P.ctuFirst[ctu], cnt = P.ctuCnt[ctu];
    // the CTU's luma origin and extent
    const int cx = (ctu % P.ctusW) << P.ctuLog2, cy = (ctu / P.ctusW) << P.ctuLog2, cw = min(ctuSize, P.W - cx), ch = min(ctuSize, P.H - cy);
    // ---- the CTU's samples, residuals and owner words -> shared memory (asynchronous 32-bit copies: the pitch is not a multiple of 16 bytes), records, flags
    for (int c = 0; c < nComp; c++) {
      const int sh = c ? 1 : 0, ox = cx >> sh, oy = cy >> sh, tw = cw >> sh, th = ch >> sh, ts = c ? V2_CS : V2_LS;
      int16_t* rec = tileRec + v2_tile_off(c); int16_t* res = tileRes + v2_tile_off(c);
      const int16_t* src = P.planes[c] + (size_t)oy * P.stride[c] + ox;
      const int16_t* rsrc = P.resi[c] ? P.resi[c] + (size_t)oy * P.stride[c] + ox : nullptr;
      if (!(P.stride[c] & 7) && !(tw & 7) && !((uintptr_t)src & 15) && !((uintptr_t)rsrc & 15)) {       // rows start on 16-byte boundaries: 8 samples per copy
        const int wv = tw >> 3, n = wv * th;
        for (int k = tid; k < n; k += V2_THREADS) {
          const int y = k / wv, x = (k - y * wv) * 8;
          cp_async16(rec + y * ts + x, src + (size_t)y * P.stride[c] + x);
          if (rsrc) cp_async16(res + y * ts + x, rsrc + (size_t)y * P.stride[c] + x);
        }
      } else {
        const int wWords = tw >> 1, n = wWords * th;
        for (int k = tid; k < n; k += V2_THREADS) {
          const int y = k / wWords, x = (k - y * wWords) * 2;
          cp_async4(rec + y * ts + x, src + (size_t)y * P.stride[c] + x);
          if (rsrc) cp_async4(res + y * ts + x, rsrc + (size_t)y * P.stride[c] + x);
        }
      }
      const int unit = c ? 2 : 4, uw = tw / unit, uh = th / unit;
      const int* osrc = P.owner[c] + (size_t)(oy / unit) * P.ownerStride[c] + ox / unit;
      for (int k = tid; k < uw * uh; k += V2_THREADS) { const int y = k / uw, x = k - y * uw; cp_async4(sown + c * 1024 + y * 32 + x, osrc + (size_t)y * P.ownerStride[c] + x); }
    }
    for (int k = tid; k < min(cnt, V2_RECS) * 4; k += V2_THREADS) cp_async4(reinterpret_cast<uint32_t*>(srec) + k, reinterpret_cast<const uint32_t*>(P.tus + first) + k);
    for (int k = tid; k < cnt; k += V2_THREADS) sflag[k] = P.compSel == 2 ? (uint8_t)(P.tus[first + k].comp == 0) : 0;      // chroma pass: the luma blocks are finished (the pass before)
    cp_async_wait_all();
    __syncthreads();

    // ---- the CTU's blocks, one group each, in decoding order
    IntraScratch& S = scratch[grp];
    // Block tickets: group g starts with block g (sNext starts past them); while a group works on a block, its lane 0 takes the group's next ticket.  Tickets
    // still go out in decoding order and only to running groups.  The ticket alternates between two words: between lane 0's write of a word and the group's
    // read of it lies the block's last barrier, and between that read and lane 0's next write of the same word the next block's first barrier.
    int slot = 0;
    for (int k = grp; k < cnt; k = S.next[slot], slot ^= 1) {
      if (lane == 0) S.next[slot] = atomicAdd(&sNext, 1);
      const int me = first + k;
      const b200_intra_tu t = k < V2_RECS ? srec[k] : P.tus[me];
      if ((P.compSel == 1 && t.comp != 0) || (P.compSel == 2 && t.comp == 0)) { intra_sync(grp + 1); continue; }      // the other channel's pass
      intra_block(P, t, me, lane, grp + 1, S, TileIo{P, tileRec, sown, sflag, first, cx, cy, cw, ch, t.comp});
      // ---- publish: the CTU's own later blocks see the tile; other CTUs read the plane, and only the samples of the CTU's last column and last row
      // (left, above and above-right references of the CTUs right of / below it): blocks that touch neither skip the done word.  After the group barrier
      // one thread releases the group's stores: at CTA scope through the done byte, at GPU scope through the done word (both cumulative over the barrier)
      intra_sync(grp + 1);
      if (lane == 0) {
        const int s = t.comp ? 1 : 0;
        __threadfence_block();
        sflag[k] = 1;
        if (t.x + (1 << t.log2w) == (cx >> s) + (cw >> s) || t.y + (1 << t.log2h) == (cy >> s) + (ch >> s)) v2_st_release(P.done + me, 1);
#ifdef B200_K6_PHASES
        k6_phases_add(1, t.comp, S.clk);
#endif
      }
    }
  }
}

// record checks of the picture path (the kernel-level wrapper checks on the host)
__global__ void __launch_bounds__(256) intra_validate_kernel(const b200_intra_tu* __restrict__ tus, int n, const b200_geom g, int* meta)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  b200_intra_tu prev;
  if (i) prev = tus[i - 1];
  if (intra_problem(tus[i], i ? &prev : nullptr, g)) atomicOr(&meta[LM_ERR], 8);
}
// K6 adds the residual plane over a whole CIIP block (resiMask 0xff).  A CIIP CU larger than the maximum transform size also covers transform units without a
// residual, where K1 writes nothing: their part of the plane must read zero, as the reference adds nothing there.  This clears every CIIP block that takes a
// residual before K1 writes the units that carry one (records are validated by then).  Few CTAs walk the whole list: most records are not CIIP.
__global__ void __launch_bounds__(128) intra_ciip_clear_kernel(const b200_intra_tu* __restrict__ tus, int numTus, int16_t* r0, int16_t* r1, int16_t* r2, int s0, int s1, int s2)
{
  for (int k = blockIdx.x; k < numTus; k += gridDim.x) {
    const b200_intra_tu t = tus[k];
    if (!t.ciip || (t.flags & B200_INTRA_ISP) || !(t.flags & B200_INTRA_ADD_RESI)) continue;
    int16_t* r = t.comp == 0 ? r0 : t.comp == 1 ? r1 : r2;
    const int s = t.comp == 0 ? s0 : t.comp == 1 ? s1 : s2, w = 1 << t.log2w, n = w << t.log2h;
    for (int i = threadIdx.x; i < n; i += blockDim.x) r[(size_t)(t.y + (i >> t.log2w)) * s + t.x + (i & (w - 1))] = 0;
  }
}

int launch_intra_ciip_clear(const b200_intra_tu* tus, size_t numTus, int16_t* const resi[3], const int stride[3], cudaStream_t s, KHook* hook)
{
  if (!numTus) return 0;
  const int grid = (int)std::min<size_t>(numTus, (size_t)2 * num_sms());
  intra_ciip_clear_kernel<<<grid, 128, 0, s>>>(tus, (int)numTus, resi[0], resi[1], resi[2], stride[0], stride[1], stride[2]); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  return 0;
}

int launch_intra_validate(const b200_intra_tu* tus, size_t numTus, const b200_geom& g, int* meta, cudaStream_t s, KHook* hook)
{
  if (!numTus) return 0;
  intra_validate_kernel<<<(unsigned)((numTus + 255) / 256), 256, 0, s>>>(tus, (int)numTus, g, meta); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  return 0;
}

// CTU-resident grid: CTAs per CTU of the widest wave-front diagonal, times 2.  Single-lane 4K I picture on an H100 80 GB HBM3 at 400 W, 128x5 groups
// (bench.py --lanes 1, I_picture_ms): 1x 10.15 ms, 1.5x 9.64, 2x 9.56, 3x 9.43, SM count (132 CTAs) 9.42 — 3x is the smallest factor that costs nothing
constexpr int kWaveCtasPerDiag2 = 6;

int launch_intra(const IntraLaunch& L, cudaStream_t s, KHook* hook)
{
  if (!L.numTus) return 0;
  hook_begin(hook, B200_KF_INTRA, s);
  IntraParams P;
  for (int c = 0; c < 3; c++) { P.planes[c] = L.planes.p[c]; P.resi[c] = L.resi[c]; P.stride[c] = L.planes.stride[c]; P.owner[c] = L.owner[c]; P.ownerStride[c] = L.ownerStride[c]; }
  if (!L.geom.chromaFormat) { P.planes[1] = P.planes[2] = nullptr; }
  P.W = L.geom.width; P.H = L.geom.height; P.bitDepth = L.geom.bitDepth; P.tus = L.tus; P.numTus = (int)L.numTus;
  P.done = L.sync; P.ticket = L.sync + L.numTus; P.err = L.sync + L.numTus + 1; P.compSel = L.compSel;
  const bool cont = L.compSel == 2;                            // second launch on the list: done words, owner maps and the processing order are kept
  if (cont) B200_CUDA(cudaMemsetAsync(P.ticket, 0, sizeof(int), s));
  else {
    B200_CUDA(cudaMemsetAsync(L.sync, 0, (L.numTus + 2) * sizeof(int), s));
    for (int c = 0; c < (L.geom.chromaFormat ? 3 : 1); c++) B200_CUDA(cudaMemsetAsync(L.owner[c], 0xff, L.ownerBytes[c], s));
  }
  P.perm = nullptr; P.ctuCnt = P.ctuFirst = P.ctuBase = nullptr;
  P.ctuLog2 = ctu_log2(L.geom); P.ctusW = (L.geom.width + L.geom.ctuSize - 1) / L.geom.ctuSize; P.ctusH = (L.geom.height + L.geom.ctuSize - 1) / L.geom.ctuSize;
  // Measurement and test switch, read on every launch (one getenv per picture): B200_INTRA_KERNEL=v1 (one CTA per block through global memory) or v2
  // (CTU-resident); unset or any other value: chosen by density.  v2 (CTU-resident) shortens the dependency chains of dense lists (I pictures); the
  // scattered intra CUs of a B picture have almost no chains and finish sooner with v1's one-CTA-per-block throughput (measured at 4K: 15 % intra CUs
  // 0.08 ms vs 0.24 ms; I picture 12.5 ms vs 8 ms).  Both launches of an LMCS two-pass picture take the same kernel: compSel 2 reuses the first one's order scratch.
  const char* variant = getenv("B200_INTRA_KERNEL");
  const bool force1 = variant && !strcmp(variant, "v1"), force2 = variant && !strcmp(variant, "v2");
  const bool dense = L.numTus >= 48 * std::max<size_t>(1, (size_t)L.geom.width * L.geom.height >> 14);                   // >= 48 blocks per 128x128 luma area
  const bool v1 = !L.order || force1 || (!force2 && !dense) || ((P.stride[0] | P.stride[1] | P.stride[2]) & 1);          // the tile loads move 32-bit words
  const unsigned grid = (unsigned)((L.numTus + 255) / 256);
  if (!cont) { intra_owner_kernel<<<(unsigned)L.numTus, 64, 0, s>>>(P); hook_count(hook); }
  if (!v1) {
    // v2: per-CTU runs of the list (decoding order keeps a CTU's blocks together), CTUs in wave-front order, one CTA per CTU at a time
    const size_t nCtu = (size_t)P.ctusW * P.ctusH;
    int* base = L.order; P.ctuCnt = base; P.ctuFirst = base + nCtu; int* ctuOrder = base + 2 * nCtu; int* counters = base + 3 * nCtu;
    if (cont) B200_CUDA(cudaMemsetAsync(counters + 1, 0, sizeof(int), s));
    else {
      B200_CUDA(cudaMemsetAsync(P.ctuCnt, 0, nCtu * sizeof(int), s));
      B200_CUDA(cudaMemsetAsync(P.ctuFirst, 0x7f, nCtu * sizeof(int), s));
      intra_ctu_count_kernel<<<grid, 256, 0, s>>>(P); hook_count(hook);
      intra_ctu_check_kernel<<<grid, 256, 0, s>>>(P); hook_count(hook);
      intra_ctu_order_kernel<<<1, 1024, nCtu * sizeof(int), s>>>(P, ctuOrder, counters); hook_count(hook);
    }
    // Grid: as many CTAs as the wave front can keep busy.  Only the CTUs of about one key x + 2 y (at most `diag` of them) run at a time — with the next
    // key's CTUs trailing them by a fraction of a CTU — and each CTA fills an SM (registers and shared memory), so a grid of SM count would hold SMs that
    // spin on done words, away from the other work of the device (the second lane's picture).  Any grid of at least one CTA is deadlock-free: CTU tickets
    // go out in wave-front order and only to running CTAs, so the oldest unfinished CTU never waits on one that has not started.
    int diag = 1;
    for (int key = 0; key < P.ctusW + 2 * P.ctusH; key++) {
      int n = 0;
      for (int y = 0; y < P.ctusH; y++) n += key - 2 * y >= 0 && key - 2 * y < P.ctusW;
      diag = std::max(diag, n);
    }
    const int ctas = (int)std::min<size_t>({nCtu, (size_t)num_sms(), (size_t)(kWaveCtasPerDiag2 * diag + 1) / 2});
    // 128x5: 96 registers, no spills (128x6 is capped at 80 and spills).  Single-lane 4K I picture, grid 2x the diagonal, H100 80 GB HBM3 at 400 W:
    // 128x5 9.56 ms, 128x6 9.99 ms
    static bool attr = false;
    if (!attr) { B200_CUDA(cudaFuncSetAttribute(intra_ctu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)V2_SMEM)); attr = true; }
    intra_ctu_kernel<<<ctas, V2_THREADS, V2_SMEM, s>>>(P, ctuOrder, counters); hook_count(hook);
    B200_CUDA(cudaGetLastError());
    hook_end(hook, B200_KF_INTRA, s);
    return 0;
  }
  const char* order = getenv("B200_INTRA_ORDER");                // measurement and test switch, read on every launch: "decode" = tickets in list order
  const bool listOrder = order && !strcmp(order, "decode");
  if (L.order && !listOrder && L.numTus >= 100 * std::max<size_t>(1, (size_t)L.geom.width * L.geom.height >> 14)) {   // >= 100 blocks per 128x128 luma area
    const size_t nCtu = (size_t)P.ctusW * P.ctusH;
    int* perm = L.order; P.ctuCnt = perm + L.numTus; P.ctuFirst = P.ctuCnt + nCtu; P.ctuBase = P.ctuFirst + nCtu;
    if (!cont) {
      B200_CUDA(cudaMemsetAsync(P.ctuCnt, 0, nCtu * sizeof(int), s));
      B200_CUDA(cudaMemsetAsync(P.ctuFirst, 0x7f, nCtu * sizeof(int), s));
      intra_ctu_count_kernel<<<grid, 256, 0, s>>>(P); hook_count(hook);
      intra_ctu_base_kernel<<<1, 1, 0, s>>>(P); hook_count(hook);
      intra_perm_kernel<<<grid, 256, 0, s>>>(P, perm); hook_count(hook);
    }
    P.perm = perm;
  }
  const int ctas = (int)std::min<size_t>(L.numTus, (size_t)num_sms() * 12);
  intra_kernel<<<ctas, IT_THREADS, 0, s>>>(P); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  hook_end(hook, B200_KF_INTRA, s);
  return 0;
}

}  // namespace b200

#ifdef B200_K6_PHASES
// the attribution build's counters: copies them to out[2][2][6] (see g_k6Phases) after the device is idle, and clears them if `reset`
extern "C" B200_API int b200_k6_phases(unsigned long long* out, int reset)
{
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, b200::g_k6Phases, sizeof(b200::g_k6Phases)) != cudaSuccess) return -1;
  if (reset) { static const unsigned long long zero[2][2][6] = {}; if (cudaMemcpyToSymbol(b200::g_k6Phases, zero, sizeof(zero)) != cudaSuccess) return -1; }
  return 0;
}
#endif
