// k1_residual.cu — K1: dequant + inverse LFNST + inverse DCT-2/DST-7/DCT-8 (+TS, BDPCM, joint CbCr)
//                  fused with the prediction add ("reco").
//
// Replaces (reference, vvdec source/Lib/CommonLib): Quant::dequant + DeQuantImpl (Quant.cpp:122-179,
// :295-381), invResDPCM (Quant.cpp:239), TrQuant::xInvLfnst / invLfnstNxNCore (TrQuant.cpp:79-106, :201-288),
// TrQuant::xIT (TrQuant.cpp:410-485) with fastInvTrans[][] / fastInvCore_ / clipCore / cpyResiClipCore
// (TrQuant_EMT.cpp:103-121, :366-405), xITransformSkip (:489), invTransformCbCr (TrQuant.cpp:108-124) and the
// reco add of DecCu::predAndReco (DecCu.cpp:455-479 -> Buffer.cpp:83 recoCore).
//
// Mapping (north_star): one thread group per TU record (a warp for TUs up to 16x16, 128 / 256 threads for 32 / 64); the TU's packed
// level corner is staged into shared memory as dequantised int16 coefficients, both 1-D stages accumulate in int32 (no tensor cores),
// stage-1 output lives in shared memory as int16 (it is clipped to 16 bit by the standard), stage-2 output goes straight to the plane.
// Both stages are 16-bit x 8-bit dot products taken two basis rows at a time (IDP.2A): the operand blocks are stored with rows k, k+1
// interleaved (one 32-bit word per pair), the cores come from kTrPair (bytes (m[k][j], m[k+1][j])), and every thread produces four
// neighbouring outputs from one operand word and one 8-byte core load per row pair.
// HBM traffic per TU = corner levels (2 B each) + 32 B record + w*h*2 B read (pred) + w*h*2 B write.
#define VVC_TABLE_QUAL static __device__ const __align__(16)
#include "vvc_tables.h"
#include "common.cuh"
#include <algorithm>

namespace b200 {

constexpr int K1_WARPS = 8;
// TU size classes (host buckets the records, order inside a picture is irrelevant: TUs never overlap):
//   class 0: w,h <= 8   class 1: <= 16   class 2: <= 32   class 3: a 64 dimension
// per warp: CB int16 dequantised coefficients (coded corner, at most min(w,32)*min(h,32)), TB int16 stage-1 output (<= min(w,32)*h)
// threads per TU: one warp for the small classes, a whole CTA for the big ones (a 64x64 TU is ~200k MACs: one warp would take >100 us)
template <int CLS> struct K1Cfg {
  static constexpr int CB = CLS == 0 ? 64 : CLS == 1 ? 256 : 1024, TB = CLS == 0 ? 64 : CLS == 1 ? 256 : CLS == 2 ? 1024 : 2048;
  static constexpr int G = CLS <= 1 ? 32 : CLS == 2 ? 128 : 256;       // group size (threads per TU)
  static constexpr int THREADS = CLS <= 1 ? K1_WARPS * 32 : G;         // big classes: exactly one group per CTA (they use __syncthreads)
  static constexpr int GROUPS = THREADS / G;                           // TUs per CTA
};

__device__ __forceinline__ const int16_t* tr_pair(int trType, int log2n)   // row-paired core (see gen_tables.cpp)
{
  const int p4 = 1 << (2 * log2n);
  if (log2n == 1) return kTrPair;                            // 2-point DCT-2 (chroma of 4-wide luma); its single pair row sits in front
  if (trType == B200_TR_DCT2) return kTrPair + 2 + (p4 - 4) / 6;
  return kTrPair + 2 + (trType == B200_TR_DCT8 ? 2730 : 3410) + (p4 - 16) / 6;
}

__device__ __forceinline__ int dequant_one(int level, int scale, int rightShift, int inMax)
{
  // Quant.cpp:146-151 / :166-171 (Intermediate_Int == int: 32-bit wrap-around arithmetic)
  const int c = clip3(-inMax - 1, inMax, level);
  int v;
  if (rightShift > 0) v = (int)((unsigned)c * (unsigned)scale + (1u << (rightShift - 1))) >> rightShift;
  else                v = (int)(((unsigned)c * (unsigned)scale) << (-rightShift));
  return clip16(v);
}

// one TU, executed by a group of G threads (`lane` = index in the group); all exits are uniform over the group
template <int CLS>
__device__ __forceinline__ void k1_tu(const b200_tu* __restrict__ tus, int t, const int16_t* __restrict__ coefs, const int32_t* __restrict__ scaling,
                                      int16_t* p0, int16_t* p1, int16_t* p2, int16_t* r0, int16_t* r1, int16_t* r2, int s0, int s1, int s2, int bitDepth, int mode,
                                      int compSel, const int* __restrict__ vpduScale, int vpduGeo, int16_t* cb, int16_t* tb, int lane)
{
  constexpr int G = K1Cfg<CLS>::G;
  auto gsync = [&]() { if (G == 32) __syncwarp(); else __syncthreads(); };

  const uint4* recp = reinterpret_cast<const uint4*>(tus + t);
  const uint4 ra = __ldg(recp), rb = __ldg(recp + 1);
  // unpack b200_tu (32 B)
  const int tx = ra.x & 0xffff, ty = ra.x >> 16;
  const int log2w = ra.y & 0xff, log2h = (ra.y >> 8) & 0xff, comp = (ra.y >> 16) & 0xff, flags = ra.y >> 24;
  int maxX = ra.z & 0xff, maxY = (ra.z >> 8) & 0xff;
  const int trType = (ra.z >> 16) & 0xff, lfnst = ra.z >> 24;
  const int ict = (int)(int8_t)(ra.w & 0xff), rightShift = (int)(int8_t)((ra.w >> 8) & 0xff);
  const int inBits = (ra.w >> 16) & 0xff, scale = ra.w >> 24;
  const unsigned coefOff = rb.x, slOff = rb.y;
  if ((compSel == 1 && comp != 0) || (compSel == 2 && comp == 0)) return;   // LMCS: luma pass / chroma pass
  if ((flags & B200_TU_RESI) && r0) { p0 = r0; p1 = r1; p2 = r2; mode = 1; }  // TU of an intra CU: residual to the residual planes, K6 reconstructs

  const int w = 1 << log2w, h = 1 << log2h;
  const int16_t* q = coefs + coefOff;
  const int qs = maxX + 1;
  const int inMax = (1 << (inBits - 1)) - 1;
  const int32_t* sl = (flags & B200_TU_SCALING) ? scaling + slOff : nullptr;
  const bool isTS = flags & B200_TU_TS;

  // coefficient tile geometry: CS = row stride of cb
  int nzW = maxX + 1, nzH = maxY + 1;
  if (lfnst && !isTS) { nzW = max(nzW, min(w, 8)); nzH = max(nzH, min(h, 8)); }
  const int CS = nzW;
  const int nzHe = (nzH + 1) & ~1;                           // rows are stored in pairs; an odd last row gets a zero partner
  auto cbi = [&](int y, int x) { return (((y >> 1) * CS + x) << 1) + (y & 1); };

  // ---- 1. dequant (Quant.cpp:295) ----
  if (flags & (B200_TU_BDPCM_H | B200_TU_BDPCM_V)) {
    // invResDPCM (Quant.cpp:239): running sum with 16-bit clip along x (H) or y (V); one lane per line.
    const bool hor = flags & B200_TU_BDPCM_H;
    const int lines = hor ? h : w, len = hor ? w : h;
    for (int l = lane; l < lines; l += G) {
      int acc = 0;
      for (int i = 0; i < len; i++) {
        const int x = hor ? i : l, y = hor ? l : i;
        const int lv = q[y * qs + x];
        acc = i ? clip16(acc + lv) : lv;
        const int sc = sl ? sl[y * w + x] * scale : scale;
        cb[cbi(y, x)] = acc ? (int16_t)dequant_one(acc, sc, rightShift, inMax) : (int16_t)0;
      }
    }
  } else {
    for (int i = lane; i < nzW * nzHe; i += G) {
      const int y = i / CS, x = i - y * CS;
      int v = 0;
      if (x <= maxX && y <= maxY) {
        const int lv = q[y * qs + x];
        if (lv) v = dequant_one(lv, sl ? sl[y * w + x] * scale : scale, rightShift, inMax);
      }
      cb[cbi(y, x)] = (int16_t)v;
    }
  }
  gsync();

  // ---- 2. inverse LFNST (TrQuant.cpp:201) ----
  if (lfnst && !isTS) {
   if (lane < 32) {     // LFNST works on 16 coefficients: the first warp of the group does it
    const int idx = (lfnst & 3) - 1, set = (lfnst >> 2) & 3, transpose = (lfnst >> 4) & 1;
    const bool big = w >= 8 && h >= 8;
    const int zo = ((w == 4 && h == 4) || (w == 8 && h == 8)) ? 8 : 16;
    int myIn = 0;
    if (lane < 16) {
      // (x,y) of diag scan pos: {0,0},{0,1},{1,0},{0,2},{1,1},{2,0},{0,3},{1,2},{2,1},{3,0},{1,3},{2,2},{3,1},{2,3},{3,2},{3,3}
      const unsigned long long XS = 0x3323213210210100ull;   // nibble i = x of scan pos i
      const unsigned long long YS = 0x3231230123012010ull;   // nibble i = y of scan pos i
      const int x = (int)((XS >> (4 * lane)) & 15), y = (int)((YS >> (4 * lane)) & 15);
      myIn = cb[cbi(y, x)];
    }
    const int8_t* m = big ? kLfnst8x8 + (set * 2 + idx) * 48 * 16 : kLfnst4x4 + (set * 2 + idx) * 16 * 16;
    const int nOut = big ? 48 : 16;
    int out0 = 0, out1 = 0;
    for (int i = 0; i < zo; i++) {
      const int v = __shfl_sync(0xffffffffu, myIn, i);
      if (lane < nOut)      out0 += v * m[lane * 16 + i];
      if (lane + 32 < nOut) out1 += v * m[(lane + 32) * 16 + i];
    }
    out0 = clip16((out0 + 64) >> 7);
    out1 = clip16((out1 + 64) >> 7);
    __syncwarp();
    // scatter (TrQuant.cpp:246-284)
    for (int r = 0; r < 2; r++) {
      const int j = lane + 32 * r;
      if (j >= nOut) break;
      const int val = r ? out1 : out0;
      int x, y;
      if (!big)        { const int a = j >> 2, b = j & 3; y = transpose ? b : a; x = transpose ? a : b; }
      else if (j < 32) { const int a = j >> 3, b = j & 7; y = transpose ? b : a; x = transpose ? a : b; }
      else             { const int k = j - 32, a = k >> 2, b = k & 3; y = transpose ? b : 4 + a; x = transpose ? 4 + a : b; }
      cb[cbi(y, x)] = (int16_t)val;
    }
   }
    maxX = max(maxX, min(w - 1, 7));
    maxY = max(maxY, min(h - 1, 7));
    gsync();
  }

  // ---- output helpers ----
  const int pmax = (1 << bitDepth) - 1;
  const int ds0 = comp == 0 ? s0 : comp == 1 ? s1 : s2;
  int16_t* dst0 = (comp == 0 ? p0 : comp == 1 ? p1 : p2) + (size_t)ty * ds0 + tx;
  const int ds1 = comp == 1 ? s2 : s1;                       // the other chroma plane (joint CbCr)
  int16_t* dst1 = ict ? (comp == 1 ? p2 : p1) + (size_t)ty * ds1 + tx : nullptr;

  // LMCS chroma residual scaling (DecCu.cpp:483 finishLMCSAndReco): scale of the VPDU that holds the TU's luma block; blocks of
  // at most 4 samples are not scaled (:506).  vpduGeo = log2(VPDU size) | VPDUs per row << 8.
  int lmScale = 0;
  if (vpduScale && comp != 0 && w * h > 4) lmScale = __ldg(vpduScale + ((ty * 2) >> (vpduGeo & 0xff)) * (vpduGeo >> 8) + ((tx * 2) >> (vpduGeo & 0xff)));
  auto emit = [&](int x, int y, int r) {
    int16_t* d = dst0 + y * ds0 + x;
    const int rs = lmScale ? lmcs_scale(r, lmScale, pmax) : r;
    *d = (int16_t)(mode == 0 ? clip3(0, pmax, *d + rs) : rs);
    if (ict) {
      // TrQuant.cpp:108-124 invTransformCbCr
      int r1 = (int)(int16_t)((ict == 2) ? r : (ict == -2) ? -r : (ict > 0) ? (r >> 1) : ((-r) >> 1));
      if (lmScale) r1 = lmcs_scale(r1, lmScale, pmax);
      int16_t* e = dst1 + y * ds1 + x;
      *e = (int16_t)(mode == 0 ? clip3(0, pmax, *e + r1) : r1);
    }
  };

  // ---- 3. transform skip (TrQuant.cpp:489) ----
  if (isTS) {
    for (int i = lane; i < w * h; i += G) {
      const int y = i >> log2w, x = i & (w - 1);
      emit(x, y, (x < nzW && y < nzH) ? (int)cb[cbi(y, x)] : 0);
    }
    return;
  }

  const int trH = trType & 3, trV = (trType >> 2) & 3;
  const int shift1 = 7, shift2 = 20 - bitDepth;

  // ---- 4. DC-only shortcut (TrQuant.cpp:429-448) ----
  if (maxX == 0 && maxY == 0 && trH == B200_TR_DCT2 && trV == B200_TR_DCT2) {
    int dc;
    if (w > 1 && h > 1) { dc = ((int)cb[0] * 64 + (1 << (shift1 - 1))) >> shift1; dc = (dc * 64 + (1 << (shift2 - 1))) >> shift2; }
    else                { dc = ((int)cb[0] * 64 + (1 << shift2)) >> (shift2 + 1); }       // one-sample-wide ISP partition: a single stage (:436)
    for (int i = lane; i < w * h; i += G) emit(i & (w - 1), i >> log2w, dc);
    return;
  }

  // ---- 5. zero-out aware extents (TrQuant.cpp:449-450) ----
  const int zoW = (trH != B200_TR_DCT2 && w == 32) ? 16 : min(w, 32);
  const int zoH = (trV != B200_TR_DCT2 && h == 32) ? 16 : min(h, 32);
  const int nCols = min(maxX + 1, zoW);   // = w - skipWidth
  const int nRows = min(maxY + 1, zoH);   // = h - skipHeight

  // ---- 5b. one-sample-wide / -high luma partitions of an ISP CU: one 1-D stage with the combined shift, no intermediate clip (TrQuant.cpp:466-482) ----
  if (w == 1 || h == 1) {
    const bool vert = w == 1;
    const int n = vert ? h : w, nIn = vert ? nRows : nCols, cstep = vert ? 1 : 2, sh = shift2 + 1;
    const int16_t* mp = tr_pair(vert ? trV : trH, vert ? log2h : log2w);
    for (int j = lane; j < n; j += G) {
      int acc = 0;
      for (int k = 0; k < nIn; k++) {
        const int mm = __ldg(mp + (k >> 1) * n + j);
        acc += (int)cb[k * cstep] * ((k & 1) ? (int)(int8_t)(mm >> 8) : (int)(int8_t)(mm & 0xff));
      }
      emit(vert ? 0 : j, vert ? j : 0, clip16((acc + (1 << (sh - 1))) >> sh));
    }
    return;
  }

  // ---- 6. stage 1: vertical, round >>7, clip to 16 bit (TrQuant_EMT.cpp:103-121, clip branch) ----
  // item = (column, group of 4 output rows); output columns are stored in pairs for stage 2; an odd last column gets a zero partner
  {
    const int16_t* mv = tr_pair(trV, log2h);
    const int nColsE = (nCols + 1) & ~1, nKp = (nRows + 1) >> 1, l2g = max(log2h - 2, 0);   // h == 2: one group, two live outputs
    for (int i = lane; i < (nColsE << l2g); i += G) {
      const int col = i >> l2g, j = (i & ((1 << l2g) - 1)) << 2;
      int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
      if (col < nCols) {
        const uint32_t* c2 = reinterpret_cast<const uint32_t*>(cb) + col;
        const uint2* m2 = reinterpret_cast<const uint2*>(mv + j);
        for (int kp = 0; kp < nKp; kp++) {
          const int a = (int)c2[kp * CS];
          const uint2 m = __ldg(m2 + ((kp << log2h) >> 2));
          a0 = __dp2a_lo(a, (int)m.x, a0); a1 = __dp2a_hi(a, (int)m.x, a1); a2 = __dp2a_lo(a, (int)m.y, a2); a3 = __dp2a_hi(a, (int)m.y, a3);
        }
      }
      int16_t* o = tb + ((((col >> 1) << log2h) + j) << 1) + (col & 1);
      o[0] = (int16_t)clip16((a0 + (1 << (shift1 - 1))) >> shift1); o[2] = (int16_t)clip16((a1 + (1 << (shift1 - 1))) >> shift1);
      if (h >= 4) { o[4] = (int16_t)clip16((a2 + (1 << (shift1 - 1))) >> shift1); o[6] = (int16_t)clip16((a3 + (1 << (shift1 - 1))) >> shift1); }
    }
  }
  gsync();

  // ---- 7. stage 2: horizontal + final round/clip (cpyResiClipCore, TrQuant_EMT.cpp:366) + reco ----
  {
    const int16_t* mh = tr_pair(trH, log2w);
    const int rnd = 1 << (shift2 - 1);
    const int nKp = (nCols + 1) >> 1, l2g = max(log2w - 2, 0);
    const uint32_t* t2 = reinterpret_cast<const uint32_t*>(tb);
    for (int i = lane; i < (h << l2g); i += G) {
      const int y = i >> l2g, x = (i & ((1 << l2g) - 1)) << 2;
      const uint2* m2 = reinterpret_cast<const uint2*>(mh + x);
      int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
      for (int kp = 0; kp < nKp; kp++) {
        const int a = (int)t2[(kp << log2h) + y];
        const uint2 m = __ldg(m2 + ((kp << log2w) >> 2));
        a0 = __dp2a_lo(a, (int)m.x, a0); a1 = __dp2a_hi(a, (int)m.x, a1); a2 = __dp2a_lo(a, (int)m.y, a2); a3 = __dp2a_hi(a, (int)m.y, a3);
      }
      emit(x, y, clip16((a0 + rnd) >> shift2)); emit(x + 1, y, clip16((a1 + rnd) >> shift2));
      if (w >= 4) { emit(x + 2, y, clip16((a2 + rnd) >> shift2)); emit(x + 3, y, clip16((a3 + rnd) >> shift2)); }
    }
  }
}

// One thread group per entry of its class's index list (the host sizes the grid from the list length it reads back after bucketing).
template <int CLS>
__global__ void __launch_bounds__(K1Cfg<CLS>::THREADS)
k1_residual_kernel(const b200_tu* __restrict__ tus, const uint32_t* __restrict__ idx, const int* __restrict__ meta, const int16_t* __restrict__ coefs,
                   const int32_t* __restrict__ scaling, int16_t* p0, int16_t* p1, int16_t* p2, int16_t* r0, int16_t* r1, int16_t* r2,
                   int s0, int s1, int s2, int bitDepth, int mode, int compSel, const int* __restrict__ vpduScale, int vpduGeo)
{
  constexpr int G = K1Cfg<CLS>::G, GROUPS = K1Cfg<CLS>::GROUPS;
  __shared__ __align__(16) int16_t s_c[GROUPS][K1Cfg<CLS>::CB];
  __shared__ __align__(16) int16_t s_t[GROUPS][K1Cfg<CLS>::TB];
  const int grp = threadIdx.x / G, lane = threadIdx.x % G;
  const int i = blockIdx.x * GROUPS + grp;
  if (i >= meta[LM_CNT + CLS]) return;                       // G == blockDim for the big classes: the whole CTA leaves together
  k1_tu<CLS>(tus, (int)idx[meta[LM_OFF + CLS] + i], coefs, scaling, p0, p1, p2, r0, r1, r2, s0, s1, s2, bitDepth, mode, compSel, vpduScale, vpduGeo, s_c[grp], s_t[grp], lane);
}

int launch_k1_residual(const K1Launch& L, StreamSet& ss, KHook* hook)
{
  if (L.numTus == 0) return 0;
  hook_begin(hook, B200_KF_K1, ss.main);
  const int vs = L.geom.ctuSize == 128 ? 64 : L.geom.ctuSize;
  int vpduGeo = 0; while ((1 << (vpduGeo + 1)) <= vs) vpduGeo++;
  vpduGeo |= ((L.geom.width + vs - 1) / vs) << 8;
  int launched = 0;
  for (int c = 3; c >= 0; c--) {          // largest TUs first: their long CTAs overlap the small classes on the other streams
    if (!L.cnt[c]) continue;
    cudaStream_t s = ss.pick(launched++);
    const int groups = c <= 1 ? K1_WARPS : 1;
    const int grid = (L.cnt[c] + groups - 1) / groups;
#define K1_GO(C) k1_residual_kernel<C><<<grid, K1Cfg<C>::THREADS, 0, s>>>(L.tus, L.idx, L.meta, L.coefs, L.scaling, L.planes.p[0], L.planes.p[1], L.planes.p[2], L.resi[0], L.resi[1], L.resi[2], \
                                                                   L.planes.stride[0], L.planes.stride[1], L.planes.stride[2], L.geom.bitDepth, L.mode, L.compSel, L.vpduScale, vpduGeo)
    switch (c) { case 0: K1_GO(0); break; case 1: K1_GO(1); break; case 2: K1_GO(2); break; default: K1_GO(3); break; }
    hook_count(hook);
#undef K1_GO
    B200_CUDA(cudaGetLastError());
  }
  ss.join();
  hook_end(hook, B200_KF_K1, ss.main);
  return 0;
}

}  // namespace b200
