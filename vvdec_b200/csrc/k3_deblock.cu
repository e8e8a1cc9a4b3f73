// k3_deblock.cu — K3: VVC deblocking, one thread per 4-sample edge segment (one 4x4 luma unit), picture-wide
//                 pass over all vertical edges, then a second launch over all horizontal edges, in place.
//
// Replaces (reference, source/Lib/CommonLib/LoopFilter.cpp): loopFilterCTU :375, xDeblockCtuArea :418,
// xEdgeFilterLuma :1463, xEdgeFilterChroma :1619, xPelFilterLumaCorePel :213, xFilteringPandQCore :129,
// xBilinearFilter :106, xPelFilterChroma :281, xUseStrongFiltering :1410, xCalcDP/DQ :1392, deriveLADFShift :1363.
//
// Why a flat pass is exact: VVC restricts filter lengths so that within one direction no edge reads a sample that
// another edge of the same direction modifies (<=4-wide blocks force length 1/1; lengths 5/7 need >=32-wide
// blocks), so all segments of a direction are independent (each side's reach: lf_sides, rules.cuh); the CPU's CTU
// wavefront (DecLibRecon.cpp:943-989) only orders V before H.  Each thread keeps one line (<=8+8 samples) in registers: decisions use lines 0 and 3, then
// the 4 lines are filtered one by one and only modified samples are stored (2-byte stores, no write-back races).
// HBM traffic: planes read+written once per direction (second pass is L2-resident at 4K) + 6 B per 4x4 unit.
#include "common.cuh"

namespace b200 {

__constant__ uint16_t c_tcTable[66] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,3,4,4,4,4,5,5,5,5,7,7,8,9,10,10,11,13,14,15,17,19,21,24,25,29,33,36,
  41,45,51,57,64,71,80,89,100,112,125,141,157,177,198,222,250,280,314,352,395 };       // H.266 Table 43 (tC')
__constant__ uint8_t c_betaTable[64] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,6,7,8,9,10,11,12,13,14,15,16,17,18,20,22,24,26,28,30,32,34,36,38,40,42,
  44,46,48,50,52,54,56,58,60,62,64,66,68,70,72,74,76,78,80,82,84,86,88 };                // H.266 Table 43 (beta')

struct LfParams {
  int16_t* plane[3];
  int stride[3];
  int W4, H4, bitDepth, ctuSize, ctuLog2, ctusW, chroma;
  const b200_lf_param* grid;
  const uint8_t* ctuSlice;      // may be null
  b200_lf_seq seq;
};

// one grid entry, fetched as three 2-byte loads (the 6-byte record is 2-byte aligned) and read by field
struct LfEdge { int qp[3], bs[3], lens; bool large; };
__device__ __forceinline__ LfEdge lf_edge(const b200_lf_param* rec)
{
  static_assert(sizeof(b200_lf_param) == 6, "b200_lf_param is fetched as three 2-byte words");
  const uint16_t* g = reinterpret_cast<const uint16_t*>(rec);
  const uint16_t w[3] = { __ldg(g), __ldg(g + 1), __ldg(g + 2) };
  b200_lf_param e;
  memcpy(&e, w, sizeof(e));
  return { { e.qp[0], e.qp[1], e.qp[2] }, { e.bs & 3, (e.bs >> 2) & 3, (e.bs >> 4) & 3 }, e.sideMaxFiltLength, ((e.flags >> 5) & 1) != 0 };
}

// one line across an edge: p[i] = i-th sample on the P side counted from the edge, q[i] likewise
struct Line { int p[8], q[8]; };

// The samples around one edge segment: line l (0..3) along the edge, sample i across it (i >= 0: q_i, i < 0: p_(-1-i)).  Every plane access of the
// kernel goes through this type, so a staged or out-of-place pass replaces it alone.
struct EdgeLines {
  int16_t* base;      // q0 of line 0
  int off, step;      // one sample across the edge, one line along it
  __device__ __forceinline__ EdgeLines(int16_t* plane, int stride, int x, int y, bool acrossX)
    : base(plane + (size_t)y * stride + x), off(acrossX ? 1 : stride), step(acrossX ? stride : 1) {}
  __device__ __forceinline__ int16_t& at(int l, int i) const { return base[l * step + i * off]; }
  __device__ __forceinline__ Line load(int l, int nP, int nQ) const   // nP / nQ samples of each side; the others read as 0
  {
    Line L;
#pragma unroll
    for (int i = 0; i < 8; i++) { L.p[i] = i < nP ? (int)at(l, -1 - i) : 0; L.q[i] = i < nQ ? (int)at(l, i) : 0; }
    return L;
  }
  __device__ __forceinline__ void put(int l, int side /*0 P,1 Q*/, int i, int oldv, int newv) const { if (newv != oldv) at(l, side ? i : -1 - i) = (int16_t)newv; }
  __device__ __forceinline__ int ladf_level() const { return (at(0, 0) + at(3, 0) + at(0, -1) + at(3, -1)) >> 2; }   // deriveLADFShift: p0, q0 of lines 0, 3
};

struct LfTcBeta { int tc, beta; };
__device__ __forceinline__ LfTcBeta lf_tc_beta(int qp, int bs, int tcOffsetDiv2, int betaOffsetDiv2, int bd)
{
  const int tc = c_tcTable[clip3(0, 65, qp + 2 * (bs - 1) + tcOffsetDiv2 * 2)];
  return { bd < 10 ? (tc + (1 << (9 - bd))) >> (10 - bd) : tc << (bd - 10), c_betaTable[clip3(0, 63, qp + betaOffsetDiv2 * 2)] << (bd - 8) };
}

// xCalcDP / xCalcDQ (LoopFilter.cpp:1392) on one side's samples a: |a2 - 2 a1 + a0|, for a large side averaged with |a5 - 2 a4 + a3|.  A chroma P
// side at a horizontal CTB boundary holds a0, a1 only: |a1 - 2 a1 + a0| (xCalcDP<true>, :1395).
__device__ __forceinline__ int side_activity(const int* a, bool large, bool chromaHorCtb = false)
{
  const int d = abs((chromaHorCtb ? a[1] : a[2]) - 2 * a[1] + a[0]);
  return large ? (d + abs(a[5] - 2 * a[4] + a[3]) + 1) >> 1 : d;
}

// one side's term of xUseStrongFiltering (LoopFilter.cpp:1410): |a3 - a0| (|a1 - a0| for chromaHorCtb), for a large side of length n = 5 or 7
// (0: not large) averaged with its far samples
__device__ __forceinline__ int side_flatness(const int* a, int n, bool chromaHorCtb)
{
  const int s = abs((chromaHorCtb ? a[1] : a[3]) - a[0]), e = n == 7 ? a[7] : a[5];
  if (!n) return s;
  return (s + (n == 7 ? abs(a[4] - a[5] - a[6] + e) : 0) + abs(a[3] - e) + 1) >> 1;
}
// xUseStrongFiltering on both decision lines (0 and 3 of a luma segment, 0 and 1 of a chroma one), each with its activity dA / dB
__device__ __forceinline__ bool strong_both(const Line& A, int dA, const Line& B, int dB, LfTcBeta t, int nP, int nQ, bool chromaHorCtb)
{
  const auto strong = [&](const Line& L, int d) {
    if (!(d < (t.beta >> 2) && abs(L.p[0] - L.q[0]) < ((t.tc * 5 + 1) >> 1))) return false;
    const int s = side_flatness(L.p, nP, chromaHorCtb) + side_flatness(L.q, nQ, false);
    return nP || nQ ? s < (t.beta * 3 >> 5) && d < (t.beta >> 4) : s < (t.beta >> 3);
  };
  return strong(A, 2 * dA) && strong(B, 2 * dB);
}

// one side (side 0 P, 1 Q) of the long filters, xFilteringPandQCore (LoopFilter.cpp:129), on line l: its n = 3, 5 or 7 samples a move towards mid
__device__ __forceinline__ void long_side(const int* a, int n, int mid, int tc, const EdgeLines& E, int l, int side)
{
  const int ref = ((n == 7 ? a[6] + a[7] : n == 5 ? a[4] + a[5] : a[2] + a[3]) + 1) >> 1;
  // coefficient / clip tables as closed forms: c7 = 59-9i, c5 = 58-13i, c3 = 53-21i ; tc7 = {6,5,4,3,2,1,1}, tc3 = {6,4,2}
#pragma unroll
  for (int i = 0; i < 7; i++)
    if (i < n) {
      const int c = n == 7 ? 59 - 9 * i : n == 5 ? 58 - 13 * i : 53 - 21 * i;
      const int t = n == 3 ? 6 - 2 * i : (i == 6 ? 1 : 6 - i);
      const int cv = (tc * t) >> 1, v = a[i];
      E.put(l, side, i, v, clip3(v - cv, v + cv, (mid * c + ref * (64 - c) + 32) >> 6));
    }
}

// long filters: xFilteringPandQCore + xBilinearFilter (LoopFilter.cpp:102-196) on one line
__device__ void filter_long(const Line& L, const EdgeLines& E, int l, int nP, int nQ, int tc)
{
  int mid;
  if (nP == nQ) {
    if (nP == 5) mid = (2 * (L.p[0] + L.q[0] + L.p[1] + L.q[1] + L.p[2] + L.q[2]) + L.p[3] + L.q[3] + L.p[4] + L.q[4] + 8) >> 4;
    else         mid = (2 * (L.p[0] + L.q[0]) + L.p[1] + L.q[1] + L.p[2] + L.q[2] + L.p[3] + L.q[3] + L.p[4] + L.q[4] + L.p[5] + L.q[5] + L.p[6] + L.q[6] + 8) >> 4;
  } else {
    const int big = max(nP, nQ), sml = min(nP, nQ);
    if (big == 7 && sml == 5) mid = (2 * (L.p[0] + L.q[0] + L.p[1] + L.q[1]) + L.p[2] + L.q[2] + L.p[3] + L.q[3] + L.p[4] + L.q[4] + L.p[5] + L.q[5] + 8) >> 4;
    else if (big == 7) {
      const int* lg = nP > nQ ? L.p : L.q; const int* sh = nP > nQ ? L.q : L.p;
      mid = (2 * (lg[0] + sh[0]) + sh[0] + 2 * (sh[1] + sh[2]) + lg[1] + sh[1] + lg[2] + lg[3] + lg[4] + lg[5] + lg[6] + 8) >> 4;
    } else mid = (L.p[0] + L.q[0] + L.p[1] + L.q[1] + L.p[2] + L.q[2] + L.p[3] + L.q[3] + 4) >> 3;
  }
  long_side(L.p, nP, mid, tc, E, l, 0);
  long_side(L.q, nQ, mid, tc, E, l, 1);
}

// xPelFilterLumaCorePel (LoopFilter.cpp:213) on line l held in registers
__device__ __forceinline__ void filter_normal(const Line& L, const EdgeLines& E, int l, int tc, bool sw, int thrCut, bool fP, bool fQ, int pmax)
{
  const int m0 = L.p[3], m1 = L.p[2], m2 = L.p[1], m3 = L.p[0], m4 = L.q[0], m5 = L.q[1], m6 = L.q[2], m7 = L.q[3];
  if (sw) {
    E.put(l, 0, 2, m1, clip3(m1 - tc, m1 + tc, (2 * m0 + 3 * m1 + m2 + m3 + m4 + 4) >> 3));
    E.put(l, 0, 1, m2, clip3(m2 - 2 * tc, m2 + 2 * tc, (m1 + m2 + m3 + m4 + 2) >> 2));
    E.put(l, 0, 0, m3, clip3(m3 - 3 * tc, m3 + 3 * tc, (m1 + 2 * m2 + 2 * m3 + 2 * m4 + m5 + 4) >> 3));
    E.put(l, 1, 0, m4, clip3(m4 - 3 * tc, m4 + 3 * tc, (m2 + 2 * m3 + 2 * m4 + 2 * m5 + m6 + 4) >> 3));
    E.put(l, 1, 1, m5, clip3(m5 - 2 * tc, m5 + 2 * tc, (m3 + m4 + m5 + m6 + 2) >> 2));
    E.put(l, 1, 2, m6, clip3(m6 - tc, m6 + tc, (m3 + m4 + m5 + 3 * m6 + 2 * m7 + 4) >> 3));
  } else {
    int delta = (9 * (m4 - m3) - 3 * (m5 - m2) + 8) >> 4;
    if (abs(delta) < thrCut) {
      delta = clip3(-tc, tc, delta);
      const int tc2 = tc >> 1;
      E.put(l, 0, 0, m3, clip3(0, pmax, m3 + delta));
      if (fP) E.put(l, 0, 1, m2, clip3(0, pmax, m2 + clip3(-tc2, tc2, ((((m1 + m3 + 1) >> 1) - m2 + delta) >> 1))));
      E.put(l, 1, 0, m4, clip3(0, pmax, m4 - delta));
      if (fQ) E.put(l, 1, 1, m5, clip3(0, pmax, m5 + clip3(-tc2, tc2, ((((m6 + m4 + 1) >> 1) - m5 - delta) >> 1))));
    }
  }
}

// xPelFilterChroma (LoopFilter.cpp:281) on line l
__device__ __forceinline__ void filter_chroma(const Line& L, const EdgeLines& E, int l, int tc, bool sw, int pmax, bool horCtb)
{
  const int m0 = L.p[3], m1 = L.p[2], m2 = L.p[1], m3 = L.p[0], m4 = L.q[0], m5 = L.q[1], m6 = L.q[2], m7 = L.q[3];
  if (sw) {
    if (horCtb) {
      E.put(l, 0, 0, m3, clip3(m3 - tc, m3 + tc, (3 * m2 + 2 * m3 + m4 + m5 + m6 + 4) >> 3));
      E.put(l, 1, 0, m4, clip3(m4 - tc, m4 + tc, (2 * m2 + m3 + 2 * m4 + m5 + m6 + m7 + 4) >> 3));
      E.put(l, 1, 1, m5, clip3(m5 - tc, m5 + tc, (m2 + m3 + m4 + 2 * m5 + m6 + 2 * m7 + 4) >> 3));
      E.put(l, 1, 2, m6, clip3(m6 - tc, m6 + tc, (m3 + m4 + m5 + 2 * m6 + 3 * m7 + 4) >> 3));
    } else {
      E.put(l, 0, 2, m1, clip3(m1 - tc, m1 + tc, (3 * m0 + 2 * m1 + m2 + m3 + m4 + 4) >> 3));
      E.put(l, 0, 1, m2, clip3(m2 - tc, m2 + tc, (2 * m0 + m1 + 2 * m2 + m3 + m4 + m5 + 4) >> 3));
      E.put(l, 0, 0, m3, clip3(m3 - tc, m3 + tc, (m0 + m1 + m2 + 2 * m3 + m4 + m5 + m6 + 4) >> 3));
      E.put(l, 1, 0, m4, clip3(m4 - tc, m4 + tc, (m1 + m2 + m3 + 2 * m4 + m5 + m6 + m7 + 4) >> 3));
      E.put(l, 1, 1, m5, clip3(m5 - tc, m5 + tc, (m2 + m3 + m4 + 2 * m5 + m6 + 2 * m7 + 4) >> 3));
      E.put(l, 1, 2, m6, clip3(m6 - tc, m6 + tc, (m3 + m4 + m5 + 2 * m6 + 3 * m7 + 4) >> 3));
    }
  } else {
    const int delta = clip3(-tc, tc, (((m4 - m3) * 4) + m2 - m5 + 4) >> 3);
    E.put(l, 0, 0, m3, clip3(0, pmax, m3 + delta));
    E.put(l, 1, 0, m4, clip3(0, pmax, m4 - delta));
  }
}

template <int DIR>   // 0: vertical edges (filter across x), 1: horizontal edges (filter across y)
__global__ void __launch_bounds__(256, 3) lf_kernel(const LfParams P, const LfSliceTab T)
{
  const int x4 = blockIdx.x * 32 + threadIdx.x, y4 = blockIdx.y * 8 + threadIdx.y;
  if (x4 >= P.W4 || y4 >= P.H4) return;
  const LfEdge e = lf_edge(P.grid + (size_t)y4 * P.W4 + x4);
  if (!(e.bs[0] | e.bs[1] | e.bs[2])) return;
  const int x = x4 * 4, y = y4 * 4;
  const b200_lf_slice& sl = T.s[P.ctuSlice ? P.ctuSlice[(y >> P.ctuLog2) * P.ctusW + (x >> P.ctuLog2)] : 0];
  if (sl.disable) return;
  const int bd = P.bitDepth, pmax = (1 << bd) - 1;

  // ------------------------------------------------------------------ luma (xEdgeFilterLuma :1463)
  if (e.bs[0]) {
    const EdgeLines E(P.plane[0], P.stride[0], x, y, DIR == 0);
    int qp = e.qp[0];
    if (P.seq.ladfEnabled) {
      int shift = P.seq.ladfQpOffset[0];
      const int lvl = E.ladf_level();
      bool go = true;
#pragma unroll
      for (int k = 1; k < 5; k++) { if (go && k < P.seq.ladfNumIntervals && lvl > P.seq.ladfIntervalLowerBound[k]) shift = P.seq.ladfQpOffset[k]; else go = false; }
      qp += shift;
    }
    const LfSides S = lf_sides(e.lens, DIR == 1 && (y & (P.ctuSize - 1)) == 0);
    const LfTcBeta t = lf_tc_beta(qp, e.bs[0], sl.tcOffsetDiv2[0], sl.betaOffsetDiv2[0], bd);
    const Line L0 = E.load(0, S.p.reads, S.q.reads), L3 = E.load(3, S.p.reads, S.q.reads);
    const int dp0 = side_activity(L0.p, false), dq0 = side_activity(L0.q, false), dp3 = side_activity(L3.p, false), dq3 = side_activity(L3.q, false);
    int mode = 0;   // 0 none, 1 normal/strong, 2 long
    bool sw = false, fP = false, fQ = false;
    if (S.p.large || S.q.large) {
      const int d0L = side_activity(L0.p, S.p.large) + side_activity(L0.q, S.q.large), d3L = side_activity(L3.p, S.p.large) + side_activity(L3.q, S.q.large);
      if (d0L + d3L < t.beta && strong_both(L0, d0L, L3, d3L, t, S.p.large ? S.p.len : 0, S.q.large ? S.q.len : 0, false)) mode = 2;
    }
    if (mode == 0 && dp0 + dq0 + dp3 + dq3 < t.beta) {
      mode = 1;
      if (S.p.len > 1 && S.q.len > 1) { const int sideThr = (t.beta + (t.beta >> 1)) >> 3; fP = (dp0 + dp3) < sideThr; fQ = (dq0 + dq3) < sideThr; }
      if (S.p.len > 2 && S.q.len > 2) sw = strong_both(L0, dp0 + dq0, L3, dp3 + dq3, t, 0, 0, false);
    }
    if (mode) {
      const int nP = mode == 2 ? S.p.reads : sw ? 4 : 3, nQ = mode == 2 ? S.q.reads : sw ? 4 : 3;   // the normal filters read p3 / q3 when strong
#pragma unroll 1
      for (int l = 0; l < 4; l++) {
        const Line L = l == 0 ? L0 : l == 3 ? L3 : E.load(l, nP, nQ);
        if (mode == 2) filter_long(L, E, l, S.p.writes, S.q.writes, t.tc);
        else           filter_normal(L, E, l, t.tc, sw, t.tc * 10, fP, fQ, pmax);
      }
    }
  }

  // ------------------------------------------------------------------ chroma 4:2:0 (xEdgeFilterChroma :1619)
  if (P.chroma && (e.bs[1] | e.bs[2]) && ((DIR == 0 ? x : y) & 15) == 0) {
    const bool horCtb = DIR == 1 && ((y >> 1) & ((P.ctuSize >> 1) - 1)) == 0;
#pragma unroll
    for (int c = 1; c <= 2; c++) {
      if (!(e.bs[c] == 2 || (e.large && e.bs[c] == 1))) continue;
      const EdgeLines E(P.plane[c], P.stride[c], x >> 1, y >> 1, DIR == 0);
      const LfTcBeta t = lf_tc_beta(e.qp[c], e.bs[c], sl.tcOffsetDiv2[c], sl.betaOffsetDiv2[c], bd);
      const Line L0 = E.load(0, horCtb ? 2 : 4, 4), L1 = E.load(1, horCtb ? 2 : 4, 4);
      bool sw = false;
      if (e.large) {
        const int d0 = side_activity(L0.p, false, horCtb) + side_activity(L0.q, false), d1 = side_activity(L1.p, false, horCtb) + side_activity(L1.q, false);
        sw = d0 + d1 < t.beta && strong_both(L0, d0, L1, d1, t, 0, 0, horCtb);
      }
      filter_chroma(L0, E, 0, t.tc, sw, pmax, horCtb);
      filter_chroma(L1, E, 1, t.tc, sw, pmax, horCtb);
    }
  }
}

int launch_lf_deblock(const LfLaunch& L, cudaStream_t s, KHook* hook)
{
  LfParams P;
  for (int c = 0; c < 3; c++) { P.plane[c] = L.planes.p[c]; P.stride[c] = L.planes.stride[c]; }
  P.W4 = (L.geom.width + 3) >> 2; P.H4 = (L.geom.height + 3) >> 2;
  P.bitDepth = L.geom.bitDepth; P.ctuSize = L.geom.ctuSize; P.ctuLog2 = ctu_log2(L.geom);
  P.ctusW = (L.geom.width + P.ctuSize - 1) >> P.ctuLog2; P.chroma = L.geom.chromaFormat == 1;
  P.ctuSlice = L.ctuSlice; P.seq = L.seq;
  const struct { void (*kernel)(LfParams, LfSliceTab); int family; const b200_lf_param* grid; } pass[2] = {
    { lf_kernel<0>, B200_KF_LF_V, L.lfV }, { lf_kernel<1>, B200_KF_LF_H, L.lfH } };
  const dim3 blk(32, 8), grd((P.W4 + 31) / 32, (P.H4 + 7) / 8);
  for (int d = 0; d < 2; d++)
    if ((L.dirs >> d) & 1) {
      hook_begin(hook, pass[d].family, s); P.grid = pass[d].grid;
      pass[d].kernel<<<grd, blk, 0, s>>>(P, L.slices);
      hook_count(hook); B200_CUDA(cudaGetLastError()); hook_end(hook, pass[d].family, s);
    }
  return 0;
}

}  // namespace b200
