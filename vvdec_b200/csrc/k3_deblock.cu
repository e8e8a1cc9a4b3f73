// k3_deblock.cu — K3: VVC deblocking, one thread per 4-sample edge segment (one 4x4 luma unit), picture-wide
//                 pass over all vertical edges, then a second launch over all horizontal edges, in place.
//
// Replaces (reference, source/Lib/CommonLib/LoopFilter.cpp): loopFilterCTU :375, xDeblockCtuArea :418,
// xEdgeFilterLuma :1463, xEdgeFilterChroma :1619, xPelFilterLumaCorePel :213, xFilteringPandQCore :129,
// xBilinearFilter :106, xPelFilterChroma :281, xUseStrongFiltering :1410, xCalcDP/DQ :1392, deriveLADFShift :1363.
//
// Why a flat pass is exact: VVC restricts filter lengths so that within one direction no edge reads a sample that
// another edge of the same direction modifies (<=4-wide blocks force length 1/1; lengths 5/7 need >=32-wide
// blocks), so all segments of a direction are independent; the CPU's CTU wavefront (DecLibRecon.cpp:943-989) only
// orders V before H.  Each thread keeps one line (<=8+8 samples) in registers: decisions use lines 0 and 3, then
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
  int W, H, W4, H4, bitDepth, ctuSize, ctuLog2, ctusW, chroma;
  const b200_lf_param* grid;
  const uint8_t* ctuSlice;      // may be null
  b200_lf_seq seq;
};

// one line across an edge: p[i] = i-th sample on the P side counted from the edge, q[i] likewise
struct Line { int p[8], q[8]; };

__device__ __forceinline__ void load_line(Line& L, const int16_t* s, int off, int nP, int nQ)
{
#pragma unroll
  for (int i = 0; i < 8; i++) { L.p[i] = i < nP ? (int)s[-(i + 1) * off] : 0; L.q[i] = i < nQ ? (int)s[i * off] : 0; }
}

__device__ __forceinline__ int dP(const Line& L, int b) { return abs(L.p[b + 2] - 2 * L.p[b + 1] + L.p[b]); }
__device__ __forceinline__ int dQ(const Line& L, int b) { return abs(L.q[b] - 2 * L.q[b + 1] + L.q[b + 2]); }
__device__ __forceinline__ int pick(const int* a, int i) { return i == 7 ? a[7] : i == 5 ? a[5] : a[3]; }

// xUseStrongFiltering (LoopFilter.cpp:1410). chromaHorCtb: P side has only 2 lines above the CTB boundary.
__device__ __forceinline__ bool use_strong(const Line& L, int d, int beta, int tc, bool largeP, bool largeQ, int maxP, int maxQ, bool chromaHorCtb)
{
  const int m3 = L.p[0], m4 = L.q[0];
  if (!(d < (beta >> 2) && abs(m3 - m4) < ((tc * 5 + 1) >> 1))) return false;
  int sp3 = chromaHorCtb ? abs(L.p[1] - m3) : abs(L.p[3] - m3);
  int sq3 = abs(L.q[3] - m4);
  if (largeP || largeQ) {
    if (largeP) {
      const int e = pick(L.p, maxP);
      if (maxP == 7) sp3 += abs(L.p[4] - L.p[5] - L.p[6] + e);
      sp3 = (sp3 + abs(L.p[3] - e) + 1) >> 1;
    }
    if (largeQ) {
      const int e = pick(L.q, maxQ);
      if (maxQ == 7) sq3 += abs(L.q[4] - L.q[5] - L.q[6] + e);
      sq3 = (sq3 + abs(e - L.q[3]) + 1) >> 1;
    }
    return (sp3 + sq3) < (beta * 3 >> 5) && d < (beta >> 4);
  }
  return (sp3 + sq3) < (beta >> 3);
}

__device__ __forceinline__ int tc_of(int idx, int bd) { return bd < 10 ? (c_tcTable[idx] + (1 << (9 - bd))) >> (10 - bd) : c_tcTable[idx] << (bd - 10); }

__device__ __forceinline__ void put(int16_t* s, int off, int side /*0 P,1 Q*/, int i, int oldv, int newv)
{
  if (newv != oldv) s[side ? i * off : -(i + 1) * off] = (int16_t)newv;
}

// long filters: xFilteringPandQCore + xBilinearFilter (LoopFilter.cpp:102-196) on one line
__device__ void filter_long(const Line& L, int16_t* s, int off, int nP, int nQ, int tc)
{
  const int refP = (L.p[nP - 1 == 6 ? 6 : nP - 1 == 4 ? 4 : 2] + pick(L.p, nP) + 1) >> 1;
  const int refQ = (L.q[nQ - 1 == 6 ? 6 : nQ - 1 == 4 ? 4 : 2] + pick(L.q, nQ) + 1) >> 1;
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
  // coefficient / clip tables as closed forms: c7 = 59-9i, c5 = 58-13i, c3 = 53-21i ; tc7 = {6,5,4,3,2,1,1}, tc3 = {6,4,2}
#pragma unroll
  for (int i = 0; i < 7; i++) {
    if (i < nP) {
      const int c = nP == 7 ? 59 - 9 * i : nP == 5 ? 58 - 13 * i : 53 - 21 * i;
      const int t = nP == 3 ? 6 - 2 * i : (i == 6 ? 1 : 6 - i);
      const int cv = (tc * t) >> 1, v = L.p[i];
      put(s, off, 0, i, v, clip3(v - cv, v + cv, (mid * c + refP * (64 - c) + 32) >> 6));
    }
    if (i < nQ) {
      const int c = nQ == 7 ? 59 - 9 * i : nQ == 5 ? 58 - 13 * i : 53 - 21 * i;
      const int t = nQ == 3 ? 6 - 2 * i : (i == 6 ? 1 : 6 - i);
      const int cv = (tc * t) >> 1, v = L.q[i];
      put(s, off, 1, i, v, clip3(v - cv, v + cv, (mid * c + refQ * (64 - c) + 32) >> 6));
    }
  }
}

// xPelFilterLumaCorePel (LoopFilter.cpp:213) on one line held in registers
__device__ __forceinline__ void filter_normal(const Line& L, int16_t* s, int off, int tc, bool sw, int thrCut, bool fP, bool fQ, int pmax)
{
  const int m0 = L.p[3], m1 = L.p[2], m2 = L.p[1], m3 = L.p[0], m4 = L.q[0], m5 = L.q[1], m6 = L.q[2], m7 = L.q[3];
  if (sw) {
    put(s, off, 0, 2, m1, clip3(m1 - tc, m1 + tc, (2 * m0 + 3 * m1 + m2 + m3 + m4 + 4) >> 3));
    put(s, off, 0, 1, m2, clip3(m2 - 2 * tc, m2 + 2 * tc, (m1 + m2 + m3 + m4 + 2) >> 2));
    put(s, off, 0, 0, m3, clip3(m3 - 3 * tc, m3 + 3 * tc, (m1 + 2 * m2 + 2 * m3 + 2 * m4 + m5 + 4) >> 3));
    put(s, off, 1, 0, m4, clip3(m4 - 3 * tc, m4 + 3 * tc, (m2 + 2 * m3 + 2 * m4 + 2 * m5 + m6 + 4) >> 3));
    put(s, off, 1, 1, m5, clip3(m5 - 2 * tc, m5 + 2 * tc, (m3 + m4 + m5 + m6 + 2) >> 2));
    put(s, off, 1, 2, m6, clip3(m6 - tc, m6 + tc, (m3 + m4 + m5 + 3 * m6 + 2 * m7 + 4) >> 3));
  } else {
    int delta = (9 * (m4 - m3) - 3 * (m5 - m2) + 8) >> 4;
    if (abs(delta) < thrCut) {
      delta = clip3(-tc, tc, delta);
      const int tc2 = tc >> 1;
      put(s, off, 0, 0, m3, clip3(0, pmax, m3 + delta));
      if (fP) put(s, off, 0, 1, m2, clip3(0, pmax, m2 + clip3(-tc2, tc2, ((((m1 + m3 + 1) >> 1) - m2 + delta) >> 1))));
      put(s, off, 1, 0, m4, clip3(0, pmax, m4 - delta));
      if (fQ) put(s, off, 1, 1, m5, clip3(0, pmax, m5 + clip3(-tc2, tc2, ((((m6 + m4 + 1) >> 1) - m5 - delta) >> 1))));
    }
  }
}

// xPelFilterChroma (LoopFilter.cpp:281)
__device__ __forceinline__ void filter_chroma(const Line& L, int16_t* s, int off, int tc, bool sw, int pmax, bool horCtb)
{
  const int m0 = L.p[3], m1 = L.p[2], m2 = L.p[1], m3 = L.p[0], m4 = L.q[0], m5 = L.q[1], m6 = L.q[2], m7 = L.q[3];
  if (sw) {
    if (horCtb) {
      put(s, off, 0, 0, m3, clip3(m3 - tc, m3 + tc, (3 * m2 + 2 * m3 + m4 + m5 + m6 + 4) >> 3));
      put(s, off, 1, 0, m4, clip3(m4 - tc, m4 + tc, (2 * m2 + m3 + 2 * m4 + m5 + m6 + m7 + 4) >> 3));
      put(s, off, 1, 1, m5, clip3(m5 - tc, m5 + tc, (m2 + m3 + m4 + 2 * m5 + m6 + 2 * m7 + 4) >> 3));
      put(s, off, 1, 2, m6, clip3(m6 - tc, m6 + tc, (m3 + m4 + m5 + 2 * m6 + 3 * m7 + 4) >> 3));
    } else {
      put(s, off, 0, 2, m1, clip3(m1 - tc, m1 + tc, (3 * m0 + 2 * m1 + m2 + m3 + m4 + 4) >> 3));
      put(s, off, 0, 1, m2, clip3(m2 - tc, m2 + tc, (2 * m0 + m1 + 2 * m2 + m3 + m4 + m5 + 4) >> 3));
      put(s, off, 0, 0, m3, clip3(m3 - tc, m3 + tc, (m0 + m1 + m2 + 2 * m3 + m4 + m5 + m6 + 4) >> 3));
      put(s, off, 1, 0, m4, clip3(m4 - tc, m4 + tc, (m1 + m2 + m3 + 2 * m4 + m5 + m6 + m7 + 4) >> 3));
      put(s, off, 1, 1, m5, clip3(m5 - tc, m5 + tc, (m2 + m3 + m4 + 2 * m5 + m6 + 2 * m7 + 4) >> 3));
      put(s, off, 1, 2, m6, clip3(m6 - tc, m6 + tc, (m3 + m4 + m5 + 2 * m6 + 3 * m7 + 4) >> 3));
    }
  } else {
    const int delta = clip3(-tc, tc, (((m4 - m3) * 4) + m2 - m5 + 4) >> 3);
    put(s, off, 0, 0, m3, clip3(0, pmax, m3 + delta));
    put(s, off, 1, 0, m4, clip3(0, pmax, m4 - delta));
  }
}

template <int DIR>   // 0: vertical edges (filter across x), 1: horizontal edges (filter across y)
__global__ void __launch_bounds__(256, 3) lf_kernel(const LfParams P, const LfSliceTab T)
{
  const int x4 = blockIdx.x * 32 + threadIdx.x, y4 = blockIdx.y * 8 + threadIdx.y;
  if (x4 >= P.W4 || y4 >= P.H4) return;
  const uint16_t* gp = reinterpret_cast<const uint16_t*>(P.grid + (size_t)y4 * P.W4 + x4);   // 6-byte record, 2-byte aligned
  const unsigned w0 = __ldg(gp), w1 = __ldg(gp + 1), w2 = __ldg(gp + 2);
  const int bsAll = (w1 >> 8) & 0x3f;
  if (!bsAll) return;
  const int x = x4 * 4, y = y4 * 4;
  const b200_lf_slice& sl = T.s[P.ctuSlice ? P.ctuSlice[(y >> P.ctuLog2) * P.ctusW + (x >> P.ctuLog2)] : 0];
  if (sl.disable) return;
  const int qpY = (int)(int8_t)(w0 & 0xff), qpU = (int)(int8_t)(w0 >> 8), qpV = (int)(int8_t)(w1 & 0xff);
  const int lens = w2 & 0xff, flags = w2 >> 8;
  const int bd = P.bitDepth, pmax = (1 << bd) - 1;

  // ------------------------------------------------------------------ luma (xEdgeFilterLuma :1463)
  const int bs = bsAll & 3;
  if (bs) {
    const int stride = P.stride[0];
    int16_t* src = P.plane[0] + (size_t)y * stride + x;
    const int off = DIR == 0 ? 1 : stride, step = DIR == 0 ? stride : 1;
    int qp = qpY;
    if (P.seq.ladfEnabled) {
      int shift = P.seq.ladfQpOffset[0];
      const int lvl = DIR == 0 ? (src[0] + src[3 * stride] + src[-1] + src[3 * stride - 1]) >> 2
                               : (src[0] + src[3] + src[-stride] + src[-stride + 3]) >> 2;
      bool go = true;
#pragma unroll
      for (int k = 1; k < 5; k++) { if (go && k < P.seq.ladfNumIntervals && lvl > P.seq.ladfIntervalLowerBound[k]) shift = P.seq.ladfQpOffset[k]; else go = false; }
      qp += shift;
    }
    const int maxP = (lens >> 4) & 7, maxQ = lens & 7;
    bool largeP = maxP > 3; const bool largeQ = maxQ > 3;
    if (DIR == 1 && (y & (P.ctuSize - 1)) == 0) largeP = false;
    const int tc = tc_of(clip3(0, 65, qp + 2 * (bs - 1) + sl.tcOffsetDiv2[0] * 2), bd);
    const int beta = c_betaTable[clip3(0, 63, qp + sl.betaOffsetDiv2[0] * 2)] << (bd - 8);
    const int nP = largeP ? maxP + 1 : 4, nQ = largeQ ? maxQ + 1 : 4;
    Line L0, L3;
    load_line(L0, src, off, nP, nQ);
    load_line(L3, src + 3 * step, off, nP, nQ);
    const int dp0 = dP(L0, 0), dq0 = dQ(L0, 0), dp3 = dP(L3, 0), dq3 = dQ(L3, 0);
    int mode = 0;   // 0 none, 1 normal/strong, 2 long
    bool sw = false, fP = false, fQ = false;
    if (largeP || largeQ) {
      const int dp0L = largeP ? (dp0 + dP(L0, 3) + 1) >> 1 : dp0, dq0L = largeQ ? (dq0 + dQ(L0, 3) + 1) >> 1 : dq0;
      const int dp3L = largeP ? (dp3 + dP(L3, 3) + 1) >> 1 : dp3, dq3L = largeQ ? (dq3 + dQ(L3, 3) + 1) >> 1 : dq3;
      const int d0L = dp0L + dq0L, d3L = dp3L + dq3L;
      if (d0L + d3L < beta && use_strong(L0, 2 * d0L, beta, tc, largeP, largeQ, maxP, maxQ, false) &&
          use_strong(L3, 2 * d3L, beta, tc, largeP, largeQ, maxP, maxQ, false)) mode = 2;
    }
    if (mode == 0 && dp0 + dq0 + dp3 + dq3 < beta) {
      mode = 1;
      if (maxP > 1 && maxQ > 1) { const int sideThr = (beta + (beta >> 1)) >> 3; fP = (dp0 + dp3) < sideThr; fQ = (dq0 + dq3) < sideThr; }
      if (maxP > 2 && maxQ > 2) sw = use_strong(L0, 2 * (dp0 + dq0), beta, tc, false, false, 7, 7, false) && use_strong(L3, 2 * (dp3 + dq3), beta, tc, false, false, 7, 7, false);
    }
    if (mode) {
#pragma unroll 1
      for (int l = 0; l < 4; l++) {
        int16_t* s = src + l * step;
        Line L;
        if (l == 0) L = L0; else if (l == 3) L = L3; else load_line(L, s, off, mode == 2 ? nP : 4, mode == 2 ? nQ : 4);
        if (mode == 2) filter_long(L, s, off, largeP ? maxP : 3, largeQ ? maxQ : 3, tc);
        else           filter_normal(L, s, off, tc, sw, tc * 10, fP, fQ, pmax);
      }
    }
  }

  // ------------------------------------------------------------------ chroma 4:2:0 (xEdgeFilterChroma :1619)
  if (P.chroma && (bsAll >> 2) && ((DIR == 0 ? x : y) & 15) == 0) {
    const int cx = x >> 1, cy = y >> 1;
    const bool horCtb = DIR == 1 && (cy & ((P.ctuSize >> 1) - 1)) == 0;
    const bool large = (flags >> 5) & 1;
#pragma unroll
    for (int c = 1; c <= 2; c++) {
      const int bsc = (bsAll >> (2 * c)) & 3;
      if (!(bsc == 2 || (large && bsc == 1))) continue;
      const int stride = P.stride[c];
      int16_t* src = P.plane[c] + (size_t)cy * stride + cx;
      const int off = DIR == 0 ? 1 : stride, step = DIR == 0 ? stride : 1;
      const int qp = c == 1 ? qpU : qpV;
      const int tc = tc_of(clip3(0, 65, qp + 2 * (bsc - 1) + (c == 1 ? sl.tcOffsetDiv2[1] : sl.tcOffsetDiv2[2]) * 2), bd);
      Line L0, L1;
      const int nP = horCtb ? 2 : 4;
      load_line(L0, src, off, nP, 4);
      load_line(L1, src + step, off, nP, 4);
      bool sw = false;
      if (large) {
        const int beta = c_betaTable[clip3(0, 63, qp + (c == 1 ? sl.betaOffsetDiv2[1] : sl.betaOffsetDiv2[2]) * 2)] * (1 << (bd - 8));
        // xCalcDP<true> (LoopFilter.cpp:1395): |p1 - 2*p1 + p0| at the horizontal CTB boundary
        const int dp0 = horCtb ? abs(L0.p[1] - 2 * L0.p[1] + L0.p[0]) : dP(L0, 0), dq0 = dQ(L0, 0);
        const int dp3 = horCtb ? abs(L1.p[1] - 2 * L1.p[1] + L1.p[0]) : dP(L1, 0), dq3 = dQ(L1, 0);
        const int d0 = dp0 + dq0, d3 = dp3 + dq3;
        if (d0 + d3 < beta) sw = use_strong(L0, 2 * d0, beta, tc, false, false, 7, 7, horCtb) && use_strong(L1, 2 * d3, beta, tc, false, false, 7, 7, horCtb);
        else { filter_chroma(L0, src, off, tc, false, pmax, horCtb); filter_chroma(L1, src + step, off, tc, false, pmax, horCtb); continue; }
      }
      filter_chroma(L0, src, off, tc, sw, pmax, horCtb);
      filter_chroma(L1, src + step, off, tc, sw, pmax, horCtb);
    }
  }
}

int launch_lf_deblock(const LfLaunch& L, cudaStream_t s, KHook* hook)
{
  LfParams P;
  for (int c = 0; c < 3; c++) { P.plane[c] = L.planes.p[c]; P.stride[c] = L.planes.stride[c]; }
  P.W = L.geom.width; P.H = L.geom.height; P.W4 = (P.W + 3) >> 2; P.H4 = (P.H + 3) >> 2;
  P.bitDepth = L.geom.bitDepth; P.ctuSize = L.geom.ctuSize; P.ctuLog2 = ctu_log2(L.geom);
  P.ctusW = (P.W + P.ctuSize - 1) >> P.ctuLog2; P.chroma = L.geom.chromaFormat == 1;
  P.ctuSlice = L.ctuSlice; P.seq = L.seq;
  dim3 blk(32, 8), grd((P.W4 + 31) / 32, (P.H4 + 7) / 8);
  if (L.dirs & 1) { hook_begin(hook, B200_KF_LF_V, s); P.grid = L.lfV; lf_kernel<0><<<grd, blk, 0, s>>>(P, L.slices); hook_count(hook); B200_CUDA(cudaGetLastError()); hook_end(hook, B200_KF_LF_V, s); }
  if (L.dirs & 2) { hook_begin(hook, B200_KF_LF_H, s); P.grid = L.lfH; lf_kernel<1><<<grd, blk, 0, s>>>(P, L.slices); hook_count(hook); B200_CUDA(cudaGetLastError()); hook_end(hook, B200_KF_LF_H, s); }
  return 0;
}

}  // namespace b200
