// affine_mv.cuh — the sub-block MVs of an affine PU record as PU::setAllAffineMv (reference CommonLib/UnitTools.cpp:2689) stores them, stated once for K2's affine
// tiles (k2_inter.cu) and the motion field of the device edge derivation (lf_derive.cuh), on the device and on the host.
#pragma once
#include <stdint.h>
#include "../../include/vvdec_b200.h"

#ifdef __CUDACC__
#define AFF_HD __host__ __device__ __forceinline__
#else
#define AFF_HD inline
#endif

namespace b200 {

AFF_HD int aff_max(int a, int b) { return a > b ? a : b; }
AFF_HD int aff_min(int a, int b) { return a < b ? a : b; }
AFF_HD int aff_log2(int v)
{
#ifdef __CUDA_ARCH__
  return 31 - __clz(v);
#else
  int l = 0; while (v > 1) { v >>= 1; l++; } return l;
#endif
}
AFF_HD void round_affine(int& x, int& y, int s) { const int o = 1 << (s - 1); x = (x + o - (x >= 0)) >> s; y = (y + o - (y >= 0)) >> s; }

// InterPrediction::isSubblockVectorSpreadOverLimit (InterPrediction.cpp:892)
AFF_HD bool spread_over_limit(int a, int b, int c, int d, int predType)
{
  const int s4 = 4 << 11, ft = 6;
  if (predType == 3) {
    int rw = aff_max(aff_max(0, 4 * a + s4), aff_max(4 * c, 4 * a + 4 * c + s4)) - aff_min(aff_min(0, 4 * a + s4), aff_min(4 * c, 4 * a + 4 * c + s4));
    int rh = aff_max(aff_max(0, 4 * b), aff_max(4 * d + s4, 4 * b + 4 * d + s4)) - aff_min(aff_min(0, 4 * b), aff_min(4 * d + s4, 4 * b + 4 * d + s4));
    rw = (rw >> 11) + ft + 3; rh = (rh >> 11) + ft + 3;
    return rw * rh > (ft + 9) * (ft + 9);
  }
  int rw = aff_max(0, 4 * a + s4) - aff_min(0, 4 * a + s4), rh = aff_max(0, 4 * b) - aff_min(0, 4 * b);
  rw = (rw >> 11) + ft + 3; rh = (rh >> 11) + ft + 3;
  if (rw * rh > (ft + 9) * (ft + 5)) return true;
  rw = aff_max(0, 4 * c) - aff_min(0, 4 * c); rh = aff_max(0, 4 * d + s4) - aff_min(0, 4 * d + s4);
  rw = (rw >> 11) + ft + 3; rh = (rh >> 11) + ft + 3;
  return rw * rh > (ft + 5) * (ft + 9);
}

struct AffModel { int LTx, LTy, dHX, dHY, dVX, dVY; bool over, prof; };

AFF_HD void aff_model(const b200_pu& pu, int l, AffModel& M)
{
  const int l2w = aff_log2(pu.w), l2h = aff_log2(pu.h);
  M.LTx = pu.mv[l][0]; M.LTy = pu.mv[l][1];
  const int RTx = pu.cpmv[l][0][0], RTy = pu.cpmv[l][0][1], LBx = pu.cpmv[l][1][0], LBy = pu.cpmv[l][1][1];
  const bool six = pu.flags & B200_PU_AFFINE6;
  M.dHX = (RTx - M.LTx) * (1 << (7 - l2w)); M.dHY = (RTy - M.LTy) * (1 << (7 - l2w));
  M.dVX = six ? (LBx - M.LTx) * (1 << (7 - l2h)) : -M.dHY; M.dVY = six ? (LBy - M.LTy) * (1 << (7 - l2h)) : M.dHX;
  M.over = spread_over_limit(M.dHX, M.dHY, M.dVX, M.dVY, pu.interDir);
  bool prof = pu.flags & (l ? B200_PU_PROF1 : B200_PU_PROF0);
  if (six ? (M.LTx == RTx && M.LTy == RTy && M.LTx == LBx && M.LTy == LBy) : (M.LTx == RTx && M.LTy == RTy)) prof = false;
  if (M.over) prof = false;
  M.prof = prof;
}

// MV of luma 4x4 sub-block (i,j) of the PU (PU::setAllAffineMv, UnitTools.cpp:2689), not yet picture-clipped
AFF_HD void aff_sub_mv(const AffModel& M, const b200_pu& pu, int i, int j, int& mx, int& my)
{
  if (M.over) { mx = M.LTx * 128 + M.dHX * (pu.w >> 1) + M.dVX * (pu.h >> 1); my = M.LTy * 128 + M.dHY * (pu.w >> 1) + M.dVY * (pu.h >> 1); }
  else        { mx = M.LTx * 128 + M.dHX * (2 + 4 * i) + M.dVX * (2 + 4 * j); my = M.LTy * 128 + M.dHY * (2 + 4 * i) + M.dVY * (2 + 4 * j); }
  round_affine(mx, my, 7);
  mx = aff_min(aff_max(mx, -(1 << 17)), (1 << 17) - 1); my = aff_min(aff_max(my, -(1 << 17)), (1 << 17) - 1);
}

}  // namespace b200
