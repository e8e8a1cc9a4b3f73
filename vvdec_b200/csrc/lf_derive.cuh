// lf_derive.cuh — the deblocking edge derivation of B200_PIC_DERIVE_LF, stated once for the device (lf_derive.cu) and the host (the glue's dry run, where it stands
// in for the device): LoopFilter::calcFilterStrengthsCTU and everything below it (reference CommonLib/LoopFilter.cpp:360-1360), on picture-wide grids instead of
// per-CTU arrays, from b200_lf_cu / b200_lf_tu records and a 4x4 motion field built from the picture's b200_pu records.
// The reference walks CU pointers (cu.left, cuP, getCU, getTU); here a CU is its record index and every such pointer is the CU that covers the position it was
// looked up for (lf_cu_at), which is what each of the reference's cached pointers is once its range check has run.
// The includer provides kGeoParams (vvc_tables.h, with the VVC_TABLE_QUAL of its side).
#pragma once
#include <stdint.h>
#include "../../include/vvdec_b200.h"
#include "affine_mv.cuh"

#ifdef __CUDACC__
#define LFD __host__ __device__ inline
#else
#define LFD inline
#endif

namespace b200 {

constexpr uint32_t LF_NONE = 0xffffffffu;
// MotionInfo of one 4x4 luma unit as far as the boundary strength reads it: per list the MV and the DPB slot of the reference picture (-1: list unused or intra)
struct LfMi { int32_t mv[2][2]; int8_t slot[2]; int8_t rsv[2]; };

struct LfDerive {
  int W4, H4;                       // grid size: 4x4 luma units = 2x2 chroma units
  int ctuSize, chroma, qpBdOffset2;
  const b200_lf_cu* cus; const b200_lf_tu* tus; const b200_pu* pus; size_t numPus;
  const uint32_t* cuMap[2];         // [H4][W4] index of the CU covering the unit, per channel type (LF_NONE: none)
  LfMi* mi;                         // [H4][W4]
  const b200_lf_slice* slices; const uint8_t* sliceB;
  b200_lf_param* grid[2];           // [H4][W4] lfV, lfH
};

struct LfArea { int x, y, w, h; };
LFD bool lf_valid(const LfArea& a) { return a.w && a.h; }
// the CU's block in channel type ch (the reference's cu.blocks[ch]; an empty area where the CU has none)
LFD bool lf_cu_has(const b200_lf_cu& c, int ch, int chroma) { return ch == c.chType || (c.chType == 0 && ch == 1 && chroma && !(c.flags & B200_LF_CU_SEP_TREE)); }
LFD LfArea lf_cu_blk(const b200_lf_cu& c, int ch, int chroma)
{
  if (ch == c.chType) return {c.x, c.y, c.w, c.h};
  if (lf_cu_has(c, ch, chroma)) return {c.x >> 1, c.y >> 1, c.w >> 1, c.h >> 1};
  return {0, 0, 0, 0};
}
LFD LfArea lf_tu_blk(const b200_lf_tu& t, int ch) { return ch ? LfArea{t.cx, t.cy, t.cw, t.ch} : LfArea{t.x, t.y, t.w, t.h}; }
template<int D> LFD int lf_perp(int x, int y) { return D ? y : x; }
template<int D> LFD int lf_parl(int x, int y) { return D ? x : y; }
template<int D> LFD int lf_perp_size(const LfArea& a) { return D ? a.h : a.w; }
template<int D> LFD int lf_parl_size(const LfArea& a) { return D ? a.w : a.h; }

// grid entry of position (x, y) in channel type ch (LoopFilterParam maps: 4x4 luma / 2x2 chroma units); -1 outside the picture
LFD int lf_unit(const LfDerive& G, int x, int y, int ch)
{
  const int s = ch ? 1 : 2;
  if (x < 0 || y < 0 || (x >> s) >= G.W4 || (y >> s) >= G.H4) return -1;
  return (y >> s) * G.W4 + (x >> s);
}
// cs.getCU( pos, ch ); `self` where no record covers the position (the records do not tile the picture: the result is then undefined, but every index stays valid)
LFD uint32_t lf_cu_at(const LfDerive& G, int x, int y, int ch, uint32_t self)
{
  const int u = lf_unit(G, x, y, ch);
  const uint32_t i = u < 0 ? LF_NONE : G.cuMap[ch][u];
  return i == LF_NONE ? self : i;
}
// getTU (LoopFilter.cpp:767), with the single-TU shortcut of its callers
LFD uint32_t lf_tu_at(const LfDerive& G, const b200_lf_cu& c, int x, int y, int ch)
{
  if (c.numTus <= 1) return c.firstTu;
  for (uint32_t k = 0; k < c.numTus; k++) {
    const LfArea b = lf_tu_blk(G.tus[c.firstTu + k], ch);
    if (b.x + b.w > x && b.y + b.h > y) return c.firstTu + k;
  }
  return c.firstTu + c.numTus - 1;
}
LFD uint32_t lf_last_tu(const b200_lf_cu& c) { return c.firstTu + (c.numTus ? c.numTus - 1 : 0); }

LFD void lf_set_edge(b200_lf_param& p, int ch, int f) { p.flags = (uint8_t)((p.flags & ~(1 << ch)) | (f << ch)); }
LFD void lf_set_cmfl(b200_lf_param& p, int f) { p.flags = (uint8_t)((p.flags & ~(1 << 5)) | (f << 5)); }
constexpr int LF_BS_TMP = 3 << 6;     // BsSet( 3, MAX_NUM_COMPONENT ): the transient bits calcFilterStrengths clears after each entry

LFD int lf_abs(int v) { return v < 0 ? -v : v; }
LFD bool lf_mv_far(const int32_t* a, const int32_t* b) { return lf_abs(a[0] - b[0]) >= 8 || lf_abs(a[1] - b[1]) >= 8; }   // nThreshold = 1/2 sample

// xGetBoundaryStrengthSingle (LoopFilter.cpp:1094-1360).  (qx, qy): position of the Q unit in the channel type of CU iq; ip: the P side's CU.
template<int D> LFD void lf_bs_single(const LfDerive& G, b200_lf_param& lfp, uint32_t iq, int qx, int qy, uint32_t ip)
{
  const b200_lf_cu& Q = G.cus[iq]; const b200_lf_cu& P = G.cus[ip];
  const int ch = Q.chType, px = qx - !D, py = qy - D;
  const b200_lf_tu& tuQ = G.tus[lf_tu_at(G, Q, qx, qy, ch)];
  const b200_lf_tu& tuP = G.tus[lf_tu_at(G, P, px, py, ch)];
  const bool hasLuma = lf_cu_has(Q, 0, G.chroma), hasChroma = G.chroma && lf_cu_has(Q, 1, G.chroma);
  const bool intraQ = Q.flags & B200_LF_CU_INTRA, intraP = P.flags & B200_LF_CU_INTRA;
  bool pcIntra = false; int chrmBS = 2;
  if (hasLuma) lfp.qp[0] = (int8_t)((Q.qp + P.qp + 1) >> 1);
  if (hasChroma) {
    const bool diff = !ch && P.treeType != 0;                       // the P side's chroma lies in another (chroma tree) CU
    const b200_lf_tu& tuQc = (Q.flags & B200_LF_CU_ISP) ? G.tus[lf_last_tu(Q)] : tuQ;
    uint32_t ipc = ip; const b200_lf_tu* tuPc = (P.flags & B200_LF_CU_ISP) ? &G.tus[lf_last_tu(P)] : &tuP;
    if (diff) { ipc = lf_cu_at(G, px >> 1, py >> 1, 1, ip); tuPc = &G.tus[lf_tu_at(G, G.cus[ipc], px >> 1, py >> 1, 1)]; }
    const b200_lf_cu& Pc = G.cus[ipc];
    pcIntra = Pc.flags & B200_LF_CU_INTRA;
    lfp.qp[1] = (int8_t)((tuPc->chromaQp[0] + tuQc.chromaQp[0] - G.qpBdOffset2 + 1) >> 1);
    lfp.qp[2] = (int8_t)((tuPc->chromaQp[1] + tuQc.chromaQp[1] - G.qpBdOffset2 + 1) >> 1);
    if (pcIntra) chrmBS = ((Pc.flags & B200_LF_CU_BDPCM_C) && intraQ && (Q.flags & B200_LF_CU_BDPCM_C)) ? 0 : 2;
  }
  const int bsMask = (hasLuma ? 3 : 0) | LF_BS_TMP | (hasChroma ? (3 << 2) | (3 << 4) : 0);
  if (intraP || intraQ) {
    const int edgeIdx = (lf_perp<D>(qx, qy) - lf_perp<D>(Q.x, Q.y)) / 4;
    const int bsY = ((P.flags & B200_LF_CU_BDPCM_Y) && (Q.flags & B200_LF_CU_BDPCM_Y)) ? 0 : 2;
    if ((Q.flags & B200_LF_CU_ISP) && edgeIdx) lfp.bs |= bsY & bsMask;
    else lfp.bs |= (bsY + (chrmBS << 2) + (chrmBS << 4)) & bsMask;
    return;
  } else if (pcIntra) lfp.bs |= (chrmBS << 2) + (chrmBS << 4);
  const bool ciip = (P.flags | Q.flags) & B200_LF_CU_CIIP;
  if ((lfp.bs & bsMask) && ciip) { lfp.bs |= (2 + (2 << 2) + (2 << 4)) & bsMask; return; }
  unsigned tmpBs = 0;
  if (lfp.bs & bsMask) {
    int cbfSum = tuQ.cbf | tuP.cbf;
    tmpBs += cbfSum & 1;
    if (!pcIntra) {                                                   // (neither P nor Q is intra here)
      const int joint = (tuQ.jointCbCr || tuP.jointCbCr) ? 1 : 0;
      cbfSum >>= 1; tmpBs += ((cbfSum & 1) | joint) << 2;
      cbfSum >>= 1; tmpBs += ((cbfSum & 1) | joint) << 4;
    }
  }
  if ((tmpBs & 3) == 1) { lfp.bs |= tmpBs & bsMask; return; }
  if (ciip) { lfp.bs |= 1 & bsMask; return; }
  if (!hasLuma) { lfp.bs |= tmpBs & bsMask; return; }
  const int tr = (lfp.bs >> 6) & 3;
  if (tr != 0 && tr != 3) { lfp.bs |= tmpBs & bsMask; return; }
  if (hasChroma) lfp.bs |= tmpBs & bsMask;
  // (P and Q are both inter here: the prediction-mode comparison at :1219 never fires without IBC)
  const int uq = lf_unit(G, qx, qy, 0), up = lf_unit(G, px, py, 0);
  if (uq < 0 || up < 0) return;
  const LfMi& mq = G.mi[uq];
  const LfMi& mp = G.mi[up];
  if (G.sliceB[Q.slice] || G.sliceB[P.slice]) {
    const int P0 = mp.slot[0], P1 = mp.slot[1], Q0 = mq.slot[0], Q1 = mq.slot[1];
    unsigned uiBs = 1;
    if ((P0 == Q0 && P1 == Q1) || (P0 == Q1 && P1 == Q0)) {
      const int32_t z[2] = {0, 0};
      const int32_t *p0 = P0 >= 0 ? mp.mv[0] : z, *p1 = P1 >= 0 ? mp.mv[1] : z, *q0 = Q0 >= 0 ? mq.mv[0] : z, *q1 = Q1 >= 0 ? mq.mv[1] : z;
      if (P0 != P1) uiBs = P0 == Q0 ? (lf_mv_far(q0, p0) || lf_mv_far(q1, p1)) : (lf_mv_far(q1, p0) || lf_mv_far(q0, p1));
      else uiBs = (lf_mv_far(q0, p0) || lf_mv_far(q1, p1)) && (lf_mv_far(q1, p0) || lf_mv_far(q0, p1));
    }
    lfp.bs |= (uiBs + tmpBs) & bsMask;
    return;
  }
  if (mp.slot[0] != mq.slot[0]) { lfp.bs |= (tmpBs + 1) & bsMask; return; }
  lfp.bs |= (lf_mv_far(mq.mv[0], mp.mv[0]) ? tmpBs + 1 : tmpBs) & bsMask;
}

// the luma filter lengths of a transform edge (:911-926, :971-984)
LFD uint8_t lf_max_len(int sizeP, int sizeQ, bool affineP)
{
  if (sizeP <= 4 || sizeQ <= 4) return 17 + 128;
  return (uint8_t)((((sizeP >= 32 ? (affineP ? 5 : 7) : 3) << 4) + (sizeQ >= 32 ? 7 : 3)) + 128);
}

// xSetMaxFilterLengthPQFromTransformSizes (LoopFilter.cpp:780-1029) for transform unit t of CU ci
template<int D> LFD void lf_tu_edges(const LfDerive& G, uint32_t ci, const b200_lf_tu& t, bool bValue, bool deriveBs, bool pqSameCtu)
{
  const b200_lf_cu& cu = G.cus[ci];
  int start = 0, end = 1;
  if (cu.flags & B200_LF_CU_SEP_TREE) { if (cu.chType == 0) end = 0; else start = 1; }
  if (start != end && (!G.chroma || !lf_valid(lf_tu_blk(t, 1)))) end = 0;
  const int cs = start != end ? 1 : 0;
  const LfArea area = lf_tu_blk(t, end), tbs = lf_tu_blk(t, start);
  const int step = D ? 1 : G.W4;                                      // OFFSET along the edge
  const bool intraQ = cu.flags & B200_LF_CU_INTRA;
  for (int ct = start; ct <= end; ct++) {
    const LfArea tb = lf_tu_blk(t, ct), cb = lf_cu_blk(cu, ct, G.chroma);
    if (!lf_valid(tb) || lf_perp<D>(tb.x, tb.y) == 0) continue;
    int gi = lf_unit(G, tb.x, tb.y, ct);
    if (gi < 0) continue;
    const int inc = ct ? 2 : 4, incFst = start ? 2 : 4;
    const bool sameCuTu = lf_perp<D>(tb.x, tb.y) == lf_perp<D>(cb.x, cb.y);
    const int sizeQ = lf_perp_size<D>(tb), len = lf_parl_size<D>(tb);
    if (ct == end && deriveBs) {
      if (start != end) {
        for (int d = 0, dFst = 0; d < len;) {
          const int qx = tb.x + D * d, qy = tb.y + (1 - D) * d, px = qx - (1 - D), py = qy - D;
          const uint32_t ip = lf_cu_at(G, px, py, ct, ci);
          const uint32_t ipf = lf_cu_at(G, D ? tbs.x + dFst : tbs.x - 1, D ? tbs.y - 1 : tbs.y + dFst, start, ci);
          const b200_lf_cu& P = G.cus[ip];
          const LfArea pb = lf_tu_blk(G.tus[lf_tu_at(G, P, px, py, ct)], ct);
          b200_lf_param& lfp = G.grid[D][gi];
          lf_set_cmfl(lfp, sizeQ >= 8 && lf_perp_size<D>(pb) >= 8);
          if (bValue) lf_bs_single<D>(G, lfp, ci, (area.x + D * d) << cs, (area.y + (1 - D) * d) << cs, ipf);
          lfp.bs &= ~LF_BS_TMP;
          if (!intraQ && !(P.flags & B200_LF_CU_INTRA) && ip == ipf && !(cu.flags & B200_LF_CU_GEO) && !(P.flags & B200_LF_CU_GEO)) {
            int distance = lf_parl<D>(pb.x, pb.y) + lf_parl_size<D>(pb) - lf_parl<D>(qx, qy);
            if (distance > len - d) distance = len - d;
            if (distance > inc && !(P.flags & (B200_LF_CU_AFFINE | B200_LF_CU_SBTMVP))) {
              const b200_lf_param param = lfp;
              for (int j = inc; j < distance; j += inc, d += inc, dFst += incFst) { gi += step; G.grid[D][gi] = param; }
            }
          }
          gi += step; d += inc; dFst += incFst;
        }
      } else {
        for (int d = 0; d < len; d += inc, gi += step) {
          const int qx = tb.x + D * d, qy = tb.y + (1 - D) * d, px = qx - (1 - D), py = qy - D;
          const uint32_t ip = lf_cu_at(G, px, py, ct, ci);
          const b200_lf_cu& P = G.cus[ip];
          const int sizeP = lf_perp_size<D>(lf_tu_blk(G.tus[lf_tu_at(G, P, px, py, ct)], ct));
          b200_lf_param& lfp = G.grid[D][gi];
          lf_set_edge(lfp, cu.chType, bValue);
          lfp.bs |= ((lfp.bs || sameCuTu) && bValue) ? LF_BS_TMP : 1 << 6;
          if (ct == 0) lfp.sideMaxFiltLength = lf_max_len(sizeP, sizeQ, P.flags & B200_LF_CU_AFFINE);
          else lf_set_cmfl(lfp, sizeQ >= 8 && sizeP >= 8);
          if (bValue) lf_bs_single<D>(G, lfp, ci, area.x + D * d, area.y + (1 - D) * d, ip);
          lfp.bs &= ~LF_BS_TMP;
        }
      }
    } else {
      for (int d = 0; d < len;) {
        const int qx = tb.x + D * d, qy = tb.y + (1 - D) * d, px = qx - (1 - D), py = qy - D;
        const uint32_t ip = lf_cu_at(G, px, py, ct, ci);
        const b200_lf_cu& P = G.cus[ip];
        const LfArea pb = lf_tu_blk(G.tus[lf_tu_at(G, P, px, py, ct)], ct);
        const int sizeP = lf_perp_size<D>(pb);
        int distance = lf_parl<D>(pb.x, pb.y) + lf_parl_size<D>(pb) - lf_parl<D>(qx, qy);
        if (distance > len - d) distance = len - d;
        if (distance < 1) distance = 1;                               // (only records whose P-side TU misses the position: keeps the walk finite)
        if (ct == 0) {
          b200_lf_param& lfp = G.grid[D][gi];
          lf_set_edge(lfp, cu.chType, bValue);
          if (bValue) {
            lfp.bs |= (lfp.bs || sameCuTu) ? LF_BS_TMP : 1 << 6;
            lfp.sideMaxFiltLength = lf_max_len(sizeP, sizeQ, P.flags & B200_LF_CU_AFFINE);
          }
          if (distance > inc) {
            const b200_lf_param tmp = lfp;
            for (int j = inc; j < distance; j += inc, d += inc) { gi += step; G.grid[D][gi] = tmp; }
          }
          d += inc; gi += step;
        } else {
          for (int j = 0; j < distance; j += inc, d += inc, gi += step) {
            b200_lf_param& lfp = G.grid[D][gi];
            if (ct == start) {
              lf_set_edge(lfp, cu.chType, bValue);
              if (bValue) lfp.bs |= (lfp.bs || sameCuTu) ? LF_BS_TMP : 1 << 6;
            }
            lf_set_cmfl(lfp, sizeQ >= 8 && sizeP >= 8);
          }
        }
      }
    }
  }
}

// xSetEdgeFilterInsidePu (:1032) for a sub-block edge of an affine / SbTMVP CU (luma)
template<int D> LFD void lf_inside_pu(const LfDerive& G, const b200_lf_cu& cu, int x, int y, int len)
{
  int gi = lf_unit(G, x, y, 0);
  if (gi < 0) return;
  for (int d = 0; d < len; d += 4, gi += D ? 1 : G.W4) {
    lf_set_edge(G.grid[D][gi], cu.chType, 1);
    if (G.grid[D][gi].bs) G.grid[D][gi].bs |= LF_BS_TMP;
  }
}

// xSetMaxFilterLengthPQForCodingSubBlocks (:707)
template<int D> LFD void lf_sub_blocks(const LfDerive& G, const b200_lf_cu& cu)
{
  const int xInc = D ? 4 : 8, yInc = D ? 8 : 4, size = D ? cu.h : cu.w, o = D ? G.W4 : 1;
  const int base = lf_unit(G, cu.x, cu.y, 0);
  if (base < 0) return;
  b200_lf_param* g = G.grid[D];
  for (int y = 0; y < cu.h; y += yInc)
    for (int x = 0; x < cu.w; x += xInc) {
      const int gi = base + (y >> 2) * G.W4 + (x >> 2), perp = D ? y : x;
      const uint8_t s = g[gi].sideMaxFiltLength;
      int maxP, maxQ, te = 0;
      if (s & 128) {
        te = 128; maxQ = (s & 7) < 5 ? (s & 7) : 5; maxP = (s >> 4) & 7;
        if (perp > 0 && maxP > 5) maxP = 5;
      } else if (perp > 0 && ((g[gi - o].sideMaxFiltLength & 128) || perp + 4 >= size || (g[gi + o].sideMaxFiltLength & 128))) maxP = maxQ = 1;
      else if (perp > 0 && (perp == 8 || (g[gi - 2 * o].sideMaxFiltLength & 128) || perp + 8 >= size || (g[gi + 2 * o].sideMaxFiltLength & 128))) maxP = maxQ = 2;
      else maxP = maxQ = 3;
      g[gi].sideMaxFiltLength = (uint8_t)((maxP << 4) + maxQ + te);
    }
}

// calcFilterStrengths (LoopFilter.cpp:495-667) for CU ci, in three parts.  First the transform edges (:543-563): the edges of one TU in one direction write
// entries of that TU's edge only, so the (TU, direction) pairs lane, lane + lanes, ... can run side by side — except in an ISP CU, whose chroma block lies in
// one TU and spans the CU: there lane d takes every TU of direction d, in order.  Returns whether the CU goes on to the sub-block edges (affine / SbTMVP) and
// the per-unit boundary strengths.
LFD bool lf_cu_tu_edges(const LfDerive& G, uint32_t ci, int lane, int lanes)
{
  const b200_lf_cu& cu = G.cus[ci];
  const int ch = cu.chType, sh = ch ? 1 : 2, mask = ~((1 << sh) - 1), ctuMask = (G.ctuSize - 1) >> ch;
  const bool refineBs = cu.flags & (B200_LF_CU_SBTMVP | B200_LF_CU_AFFINE | B200_LF_CU_ISP);
  const bool pqCuSameCtuHor = (cu.y & ctuMask) > 0, pqCuSameCtuVer = (cu.x & ctuMask) > 0;
  const bool isp = cu.flags & B200_LF_CU_ISP;
  for (int k = isp ? (lanes == 1 ? 0 : (lane < 2 ? lane : 2 * cu.numTus)) : lane; k < 2 * (int)cu.numTus; k += isp && lanes > 1 ? 2 : lanes) {
    const b200_lf_tu& t = G.tus[cu.firstTu + (k >> 1)];
    const LfArea tb = lf_tu_blk(t, ch);
    const bool atLeft = (tb.x & mask) == cu.x, atTop = (tb.y & mask) == cu.y;
    if (!(k & 1)) lf_tu_edges<0>(G, ci, t, atLeft ? (cu.flags & B200_LF_CU_AVAIL_LEFT) != 0 : true, !refineBs, atLeft ? pqCuSameCtuVer : true);
    else          lf_tu_edges<1>(G, ci, t, atTop ? (cu.flags & B200_LF_CU_AVAIL_TOP) != 0 : true, !refineBs, atTop ? pqCuSameCtuHor : true);
  }
  return refineBs;
}
// ... then, of an affine or SbTMVP CU (luma, single tree), the 8x8 sub-block edges of direction D (:567-604), which read the filter lengths the transform
// edges of that direction left ...
template<int D> LFD void lf_cu_sub_block_edges(const LfDerive& G, uint32_t ci)
{
  const b200_lf_cu& cu = G.cus[ci];
  if (!(cu.flags & (B200_LF_CU_SBTMVP | B200_LF_CU_AFFINE))) return;
  for (int off = 8; off < (D ? cu.h : cu.w); off += 8) lf_inside_pu<D>(G, cu, D ? cu.x : cu.x + off, D ? cu.y + off : cu.y, D ? cu.w : cu.h);
  lf_sub_blocks<D>(G, cu);
}
// ... and last (:611-666) every unit of the CU whose edge is on gets its boundary strength, and the transient bits go.  Each entry is on its own: units
// lane, lane + lanes, ... of each direction (the device spreads a CU's units over a warp).
LFD void lf_cu_bs_walk(const LfDerive& G, uint32_t ci, int lane, int lanes)
{
  const b200_lf_cu& cu = G.cus[ci];
  const int ch = cu.chType, pel = ch ? 2 : 4, nx = cu.w / pel, n = nx * (cu.h / pel);
  for (int k = lane; k < n; k += lanes) {
    const int x = (k % nx) * pel, y = (k / nx) * pel;
    const int gi = lf_unit(G, cu.x + x, cu.y + y, ch);
    if (gi < 0) continue;
    b200_lf_param& lfp = G.grid[0][gi];
    if ((lfp.flags >> ch) & 1) lf_bs_single<0>(G, lfp, ci, cu.x + x, cu.y + y, x ? ci : lf_cu_at(G, cu.x - 1, cu.y + y, ch, ci));
    lfp.bs &= ~LF_BS_TMP;
  }
  for (int k = lane; k < n; k += lanes) {
    const int x = (k % nx) * pel, y = (k / nx) * pel;
    const int gi = lf_unit(G, cu.x + x, cu.y + y, ch);
    if (gi < 0) continue;
    b200_lf_param& lfp = G.grid[1][gi];
    if ((lfp.flags >> ch) & 1) lf_bs_single<1>(G, lfp, ci, cu.x + x, cu.y + y, y ? ci : lf_cu_at(G, cu.x + x, cu.y - 1, ch, ci));
    lfp.bs &= ~LF_BS_TMP;
  }
}

// calcFilterStrengthsCTU (:360) walks a CTU's CUs in decoding order and returns at the first CU of a slice with deblocking disabled.  Here the CUs run one
// by one, in any order within one channel type: a CU writes grid entries of its own blocks only and reads no entry another CU of its channel
// type writes.  A chroma-tree CU reads what the luma CUs of its area left (the Bs of their edges), so chroma-tree CUs go after every luma-type CU — as in
// the reference, where a CTU's chroma tree follows the luma tree of the same area.  ctuCus: the CTU ranges; anyDisabled: some slice has deblocking off
// (then the CU runs only if no CU before it in its CTU, itself included, is in such a slice).
LFD bool lf_cu_runs(const LfDerive& G, uint32_t ci, const uint32_t* ctuCus, int nCtu, bool anyDisabled)
{
  if (!anyDisabled) return true;
  int lo = 0, hi = nCtu - 1;                                          // the CTU whose range holds ci
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (ctuCus[mid] <= ci) lo = mid; else hi = mid - 1; }
  for (uint32_t k = ctuCus[lo]; k <= ci; k++) if (G.slices[G.cus[k].slice].disable) return false;
  return true;
}

// ---- the CU maps and the motion field ----
// cs.getCU's maps: every unit of the CU's block in each channel type it has
// (units lane, lane + lanes, ... of each block)
LFD void lf_map_cu(const LfDerive& G, uint32_t* const map[2], uint32_t ci, int lane, int lanes)
{
  const b200_lf_cu& cu = G.cus[ci];
  for (int ch = 0; ch < 2; ch++) {
    if (!lf_cu_has(cu, ch, G.chroma)) continue;
    const LfArea b = lf_cu_blk(cu, ch, G.chroma); const int s = ch ? 1 : 2;
    const int x0 = b.x >> s, y0 = b.y >> s, nx = ((b.x + b.w + (1 << s) - 1) >> s) - x0, n = nx * (((b.y + b.h + (1 << s) - 1) >> s) - y0);
    for (int k = lane; k < n; k += lanes) {
      const int x = x0 + k % nx, y = y0 + k / nx;
      if (x < G.W4 && y < G.H4) map[ch][y * G.W4 + x] = ci;
    }
  }
}

// the spec's disLut (= g_Dis, Rom.cpp:593)
LFD int lf_geo_dis(int i)
{
  const int base[9] = {8, 8, 8, 8, 4, 4, 2, 1, 0};
  i &= 31;
  return i <= 8 ? base[i] : i <= 16 ? -base[16 - i] : i <= 24 ? -base[i - 16] : base[32 - i];
}

// What MIDER leaves in the motion field for the units of one PU record of CU cu (before DMVR): the record's lists (a list the CU uses whose slot the record
// dropped — xCheckIdenticalMotion — is the other list's picture), affine sub-block MVs as PU::setAllAffineMv (UnitTools.cpp:2689), GEO as PU::spanGeoMotionInfo
// (:3184).  geoParams: kGeoParams.
LFD void lf_pu_motion(const LfDerive& G, const b200_lf_cu& cu, const b200_pu& p, const int16_t* geoParams, int lane, int lanes)
{
  const int x0 = p.x >> 2, y0 = p.y >> 2, nx = p.w >> 2, ny = p.h >> 2;
  if (cu.flags & B200_LF_CU_GEO) {
    const int split = (uint8_t)p.bcwW1 & 63, angle = geoParams[split * 2], distIdx = geoParams[split * 2 + 1];
    const bool flip = angle >= 13 && angle <= 27;
    const int dX = angle, dY = (angle + 8) % 32;
    int offX = -(int)p.w >> 1, offY = -(int)p.h >> 1;
    if (distIdx > 0) {
      if (angle % 16 == 8 || (angle % 16 != 0 && p.h >= p.w)) offY += angle < 16 ? ((distIdx * p.h) >> 3) : -((distIdx * p.h) >> 3);
      else offX += angle < 16 ? ((distIdx * p.w) >> 3) : -((distIdx * p.w) >> 3);
    }
    const int l0 = cu.geoLists & 1, l1 = (cu.geoLists >> 1) & 1;
    LfMi part[3];
    for (int q = 0; q < 2; q++) {
      const int l = q ? l1 : l0;
      part[q].slot[l] = p.refSlot[q]; part[q].slot[1 - l] = -1;
      part[q].mv[l][0] = p.mv[q][0]; part[q].mv[l][1] = p.mv[q][1]; part[q].mv[1 - l][0] = part[q].mv[1 - l][1] = 0;
    }
    if (l0 != l1) {                                                   // the blend region holds both: list 0 from the partition that predicts from list 0
      const int a = l0 == 0 ? 0 : 1;
      part[2].slot[0] = p.refSlot[a]; part[2].mv[0][0] = p.mv[a][0]; part[2].mv[0][1] = p.mv[a][1];
      part[2].slot[1] = p.refSlot[1 - a]; part[2].mv[1][0] = p.mv[1 - a][0]; part[2].mv[1][1] = p.mv[1 - a][1];
    } else part[2] = part[1];
    for (int k = lane; k < nx * ny; k += lanes) {
      const int x = k % nx, y = k / nx;
      const int motionIdx = (((4 * x + offX) * 2) + 5) * lf_geo_dis(dX) + (((4 * y + offY) * 2) + 5) * lf_geo_dis(dY);
      const int m = lf_abs(motionIdx) < 32 ? 2 : (motionIdx <= 0 ? 1 - flip : flip);
      if (y0 + y < G.H4 && x0 + x < G.W4) G.mi[(y0 + y) * G.W4 + x0 + x] = part[m];
    }
    return;
  }
  AffModel M[2];
  for (int l = 0; l < 2; l++) if (p.flags & B200_PU_AFFINE) aff_model(p, l, M[l]);
  for (int k = lane; k < nx * ny; k += lanes) {
      const int x = k % nx, y = k / nx;
      if (y0 + y >= G.H4 || x0 + x >= G.W4) continue;
      LfMi m;
      for (int l = 0; l < 2; l++) {
        const bool used = (p.interDir >> l) & 1;
        m.slot[l] = used ? (p.refSlot[l] >= 0 ? p.refSlot[l] : p.refSlot[1 - l]) : -1;
        int mx = 0, my = 0;
        if (used) { if (p.flags & B200_PU_AFFINE) aff_sub_mv(M[l], p, x, y, mx, my); else { mx = p.mv[l][0]; my = p.mv[l][1]; } }
        m.mv[l][0] = mx; m.mv[l][1] = my;
      }
      m.rsv[0] = m.rsv[1] = 0;
      G.mi[(y0 + y) * G.W4 + x0 + x] = m;
  }
}

// the motion field of inter CU ci: its PU records (one, or the SbTMVP runs that tile it) in order from firstPu
LFD void lf_cu_motion(const LfDerive& G, uint32_t ci, const int16_t* geoParams, int lane, int lanes)
{
  const b200_lf_cu& cu = G.cus[ci];
  if ((cu.flags & B200_LF_CU_INTRA) || cu.chType) return;
  const int area = cu.w * cu.h;
  int covered = 0;
  for (size_t k = cu.firstPu; k < G.numPus && covered < area; k++) {
    lf_pu_motion(G, cu, G.pus[k], geoParams, lane, lanes);
    covered += G.pus[k].w * G.pus[k].h;
  }
}

// The whole derivation on one thread, in the order the device kernels keep (CU maps, motion field, luma-type CUs, chroma-tree CUs): what the glue runs in
// place of the device when it has none, and what the CPU tests compile.  G's maps, motion field and grids are cleared here.
inline void lf_derive_serial(const LfDerive& G, uint32_t* const map[2], size_t numCus, const uint32_t* ctuCus, int nCtu, const int16_t* geoParams)
{
  const size_t n4 = (size_t)G.W4 * G.H4;
  for (size_t u = 0; u < n4; u++) { map[0][u] = map[1][u] = LF_NONE; G.mi[u] = LfMi{}; G.grid[0][u] = G.grid[1][u] = b200_lf_param{}; }
  bool anyDisabled = false;
  for (uint32_t ci = 0; ci < numCus; ci++) anyDisabled = anyDisabled || G.slices[G.cus[ci].slice].disable;
  for (uint32_t ci = 0; ci < numCus; ci++) lf_map_cu(G, map, ci, 0, 1);
  for (uint32_t ci = 0; ci < numCus; ci++) lf_cu_motion(G, ci, geoParams, 0, 1);
  for (int ch = 0; ch < 2; ch++)
    for (uint32_t ci = 0; ci < numCus; ci++)
      if (G.cus[ci].chType == ch && lf_cu_runs(G, ci, ctuCus, nCtu, anyDisabled) && lf_cu_tu_edges(G, ci, 0, 1)) {
        lf_cu_sub_block_edges<0>(G, ci); lf_cu_sub_block_edges<1>(G, ci); lf_cu_bs_walk(G, ci, 0, 1);
      }
}

}  // namespace b200
