// k5_alf.cu — K5: adaptive loop filter. Luma: one CTA per 32x32 block (the reference's classification block): the block
// plus a 4-sample halo is staged in shared memory, 4 threads per 4x4 block compute the Laplacian sums (warp-shuffle reduce), then every thread filters 4 samples with
// the 7x7 diamond, two output samples per 32-bit lane: packed 16-bit subtract / clamp (VIADD.16x2, VIMNMX.S16x2) and a
// 16x8-bit dot product per tap (IDP.2A); coefficients outside int8 (only +128 is legal) fall back to scalar arithmetic.  Chroma: one thread per 4 samples does the 5x5 diamond and adds CC-ALF from the pre-ALF luma.
//
// Which sample a tap reads is decided in two places only: AlfView says where a sample of a plane comes from (the CTU's clipped sides and padded corners,
// else the picture's border extension), and the reach functions below say how far a row may reach across the CTU's virtual boundary.  An explicit virtual
// boundary (SPS / picture header) would be one more rule in each.  Each diamond's tap geometry is stated once (ALF7, ALF5), and the chroma kernel fetches
// every row, chroma or luma, through alf_window.
// Every plane K5 reads starts on a 256-byte boundary (pic_planes) with a stride of a multiple of 4 samples (both entry points check geom_problem(.., 4)),
// so rows move 8 bytes at a time wherever they lie inside the picture; and ALF is refused above 10 bit, so a packed half (a sum of two clipped differences,
// at most 2 * 2^bd) fits 16 bit.
//
// Replaces (reference, source/Lib/CommonLib/AdaptiveLoopFilter.cpp): processCTU :466, filterCTU :664 (!isCrssByVBs
// path), filterAreaLuma :498, deriveClassificationBlk :969, filterBlk<ALF_FILTER_7|5> :1175, filterAreaChroma :546,
// filterBlkCcAlf :1348, filterBlkCcAlfBoth :1447, prepareCTU :453.
// HBM traffic: S*2 B read + S*2 B written (+ halo re-reads served by L2) + 8 B/CTU + filter tables once.
#include "common.cuh"

namespace b200 {

constexpr int TB = 32;            // tile (block) size
constexpr int HALO = 4;
constexpr int TS = TB + 2 * HALO; // 40
constexpr int TSW = 44;           // shared row stride in samples (88 B: every row is 8-byte aligned)

struct AlfParams {
  const int16_t* src[3]; int16_t* dst[3]; int stride[3];
  int W, H, bitDepth, ctuSize, ctuLog2, ctusW;
  const b200_alf_ctu* ctus;
  const int16_t *lumaCoeff, *lumaClip, *chromaCoeff, *chromaClip, *cc0, *cc1;
};

// One component plane as the filters of one CTU read it: where the sample at (x, y) comes from.  (x0, y0)-(x1, y1): the CTU in the plane's samples;
// f: b200_alf_ctu::enable[0] bits 1..6, the CTU's sides that may not be read and its padded corners (include/vvdec_b200.h); pm: 0, or 2 for a chroma
// plane padded with the luma margin (B200_ALF_PAD_WIDE).  Without flags a position outside the picture reads the nearest sample inside.
struct AlfView {
  const int16_t* p; int stride, W, H, x0, y0, x1, y1, f, pm;
  __device__ const int16_t* row(int y) const { return p + (size_t)min(max(y, 0), H - 1) * stride; }
  __device__ int at(int x, int y) const
  {
    if (!f) return row(y)[min(max(x, 0), W - 1)];
    if ((f & B200_ALF_PAD_TL) && x < x0 + pm && y < y0 + pm) x = x0 + pm;             // raster-slice corners: the row's sample of the CTU's first / last column
    else if ((f & B200_ALF_PAD_BR) && x > x1 - pm && y > y1 - pm) x = x1 - pm;
    x = min(max(x, (f & B200_ALF_CLIP_LEFT) ? x0 : 0), (f & B200_ALF_CLIP_RIGHT) ? x1 : W - 1);
    y = min(max(y, (f & B200_ALF_CLIP_TOP) ? y0 : 0), (f & B200_ALF_CLIP_BOTTOM) ? y1 : H - 1);
    return p[(size_t)y * stride + x];
  }
};
// The view of a W x H plane for the CTU that holds (x, y); l2: log2 of the CTU size in the plane's samples.  CC-ALF's luma view is the luma plane's view at
// the chroma position doubled: the chroma CTU doubled, clipped to the luma picture.
__device__ __forceinline__ AlfView alf_view(const int16_t* p, int stride, int W, int H, int l2, int x, int y, int f, int pm)
{
  AlfView v; v.p = p; v.stride = stride; v.W = W; v.H = H; v.f = f; v.pm = pm;
  v.x0 = (x >> l2) << l2; v.y0 = (y >> l2) << l2; v.x1 = min(v.x0 + (1 << l2), W) - 1; v.y1 = min(v.y0 + (1 << l2), H) - 1;
  return v;
}

// ---- the CTU's virtual boundary (the reference's line buffer, :407-411): vbPos = CTU height - 4 luma rows, - 2 chroma rows.  No filter reads across it;
// each rule is a function of the row's position p in its CTU (p = y & (CTU height - 1)). ----
// Classification, row pairs (deriveClassificationBlk :1002-1010): the pair starting at picture row gy reads rows gy + up .. gy + dn; the pair 2 rows above
// the boundary stops at its own second row, the pair starting on it starts at its own first row.
__device__ __forceinline__ void alf_class_rows(int gy, int vbH, int vbPos, int& up, int& dn)
{
  up = -1; dn = 2;
  if (gy > 0 && (gy & (vbH - 1)) == vbPos - 2) dn = 1;
  else if (gy > 0 && (gy & (vbH - 1)) == vbPos) up = 0;
}
// Classification, 4x4 blocks (:1076-1100): the block starting 4 rows above the boundary drops its last row pair (r = 3), the block starting on it its
// first (r = 0); both weigh their activity by 3/2.  Returns 1 above, 2 on the boundary, else 0.
__device__ __forceinline__ int alf_class_vb(int y0, int vbH, int vbPos) { const int p = y0 & (vbH - 1); return p == vbPos - 4 ? 1 : p == vbPos ? 2 : 0; }
// The 7x7 (r = 3) and 5x5 (r = 2) diamonds (filterBlk :1260-1282): rows up to min(r, the rows left before the boundary) above and below, the same number
// on both sides.  The rows next to it (reach 0) round their sum with 3 more bits (:1313).
__device__ __forceinline__ int alf_reach(int p, int vbPos, int r) { return min(r, p < vbPos ? vbPos - 1 - p : p - vbPos); }
// CC-ALF (filterBlkCcAlf :1401-1414): the chroma row at luma row p reads luma rows p + o2, p, p + o1, p + o3.
__device__ __forceinline__ void ccalf_rows(int p, int vbPos, int& o1, int& o2, int& o3)
{
  o1 = 1; o2 = -1; o3 = 2;
  if (p == vbPos - 2 || p == vbPos + 1) o3 = 1;
  else if (p == vbPos - 1 || p == vbPos) o1 = o2 = o3 = 0;
}

// The diamonds' taps (filterBlk :1175): tap n weighs the clipped differences of the samples at (dy, dx) and (-dy, -dx) from the centre
struct AlfTap { int dy, dx; };
__device__ constexpr AlfTap ALF7[12] = {{3, 0}, {2, 1}, {2, 0}, {2, -1}, {1, 2}, {1, 1}, {1, 0}, {1, -1}, {1, -2}, {0, 3}, {0, 2}, {0, 1}};
__device__ constexpr AlfTap ALF5[6] = {{2, 0}, {1, 1}, {1, 0}, {1, -1}, {0, 2}, {0, 1}};

__device__ __forceinline__ int clipd(int c, int ref, int a, int b) { return clip3(-c, c, a - ref) + clip3(-c, c, b - ref); }
// The two samples at offset j (compile time) of a row held as sample pairs from offset -4: odd offsets are built with one byte-permute from two neighbours
__device__ __forceinline__ uint32_t alf_pair(const uint32_t* w, int j) { return (j & 1) ? __byte_perm(w[(j + 3) >> 1], w[(j + 5) >> 1], 0x5432) : w[(j + 4) >> 1]; }

// Samples x + O .. x + O + N - 1 of row y of a view into w.  An inner thread (the 4-sample groups the window touches lie inside the picture, and the CTU
// has no flags) loads each group the window takes two or more samples of as one 8-byte vector, and a lone sample by itself; other threads read sample by
// sample through the view.
template <int O, int N> __device__ __forceinline__ void alf_window(const AlfView& v, int x, int y, bool inner, int* w)
{
  if (inner) {
    const int16_t* q = v.row(y) + x;
#pragma unroll
    for (int g = O & ~3; g < O + N; g += 4) {
      const int lo = max(g, O), hi = min(g + 4, O + N);
      if (hi - lo == 1) { w[lo - O] = q[lo]; continue; }
      int s[4]; unpack4(__ldg(reinterpret_cast<const uint2*>(q + g)), s);
#pragma unroll
      for (int k = lo; k < hi; k++) w[k - O] = s[k - g];
    }
  } else {
#pragma unroll
    for (int k = 0; k < N; k++) w[k] = v.at(x + O + k, y);
  }
}

__global__ void __launch_bounds__(256) alf_luma_kernel(const AlfParams P)
{
  __shared__ __align__(16) int16_t t[TS][TSW];
  __shared__ uint16_t s_cls[64];
  const int bx0 = blockIdx.x * TB, by0 = blockIdx.y * TB;
  const int tid = threadIdx.x;
  const b200_alf_ctu cp = P.ctus[(by0 >> P.ctuLog2) * P.ctusW + (bx0 >> P.ctuLog2)];
  const int stride = P.stride[0];
  const int bw = min(TB, P.W - bx0), bh = min(TB, P.H - by0);

  if (!(cp.enable[0] & 1)) {   // unfiltered CTUs are copied (AdaptiveLoopFilter.cpp:717)
    for (int i = tid; i < bh * (bw >> 2); i += 256) {
      const int y = i / (bw >> 2), x = (i - y * (bw >> 2)) * 4;
      *reinterpret_cast<uint2*>(P.dst[0] + (size_t)(by0 + y) * stride + bx0 + x) = *reinterpret_cast<const uint2*>(P.src[0] + (size_t)(by0 + y) * stride + bx0 + x);
    }
    return;
  }

  // ---- stage tile + halo ----
  const AlfView v = alf_view(P.src[0], stride, P.W, P.H, P.ctuLog2, bx0, by0, cp.enable[0] & ~1, 0);
  if (!v.f && bx0 >= HALO && bx0 + TB + HALO <= P.W && by0 >= HALO && by0 + TB + HALO <= P.H) {
    const int16_t* s0 = P.src[0] + (size_t)(by0 - HALO) * stride + bx0 - HALO;      // interior tile: 40 rows x 10 8-byte words
    for (int i = tid; i < TS * (TS / 4); i += 256) {
      const int ty = i / (TS / 4), c = i - ty * (TS / 4);
      cp_async8(&t[ty][c * 4], reinterpret_cast<const uint2*>(s0 + (size_t)ty * stride) + c);
    }
    cp_async_wait_all();
  } else {                                                  // picture edges, clipped CTU sides, padded corners (filterCTU :763-848)
    for (int i = tid; i < TS * TS; i += 256) {
      const int ty = i / TS, tx = i - ty * TS;
      t[ty][tx] = v.at(bx0 + tx - HALO, by0 + ty - HALO);
    }
  }
  __syncthreads();

  const int vbH = P.ctuSize, vbPos = P.ctuSize - 4;

  // ---- classification (AdaptiveLoopFilter.cpp:969): thread = (4x4 block b, row pair r) ----
  {
    const int b = tid >> 2, r = tid & 3;
    const int bxi = b & 7, byi = b >> 3;
    const int y0 = by0 + byi * 4, x0l = bxi * 4;              // block origin: global y, tile-local x
    const int vb = alf_class_vb(y0, vbH, vbPos);
    int sV = 0, sH = 0, sD0 = 0, sD1 = 0;
    if (!((vb == 1 && r == 3) || (vb == 2 && r == 0))) {
      const int gy = y0 - 2 + 2 * r;                          // first row of the pair (global)
      const int ly = byi * 4 - 2 + 2 * r + HALO;              // tile row
      int up, dn2;
      alf_class_rows(gy, vbH, vbPos, up, dn2);
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const int lx = x0l - 2 + 2 * c + HALO;
        const int a = t[ly][lx] << 1, bb = t[ly + 1][lx + 1] << 1;
        sV  += abs(a - t[ly + up][lx] - t[ly + 1][lx])          + abs(bb - t[ly][lx + 1] - t[ly + dn2][lx + 1]);
        sH  += abs(a - t[ly][lx + 1] - t[ly][lx - 1])           + abs(bb - t[ly + 1][lx + 2] - t[ly + 1][lx]);
        sD0 += abs(a - t[ly + up][lx - 1] - t[ly + 1][lx + 1])  + abs(bb - t[ly][lx] - t[ly + dn2][lx + 2]);
        sD1 += abs(a - t[ly + 1][lx - 1] - t[ly + up][lx + 1])  + abs(bb - t[ly + dn2][lx] - t[ly][lx + 2]);
      }
    }
#pragma unroll
    for (int m = 1; m < 4; m <<= 1) {
      sV += __shfl_xor_sync(0xffffffffu, sV, m); sH += __shfl_xor_sync(0xffffffffu, sH, m);
      sD0 += __shfl_xor_sync(0xffffffffu, sD0, m); sD1 += __shfl_xor_sync(0xffffffffu, sD1, m);
    }
    if (r == 0) {
      const int shift = P.bitDepth + 4;
      const int act = clip3(0, 15, ((sV + sH) * (vb ? 96 : 64)) >> shift);
      const unsigned long long TH = 0x4333333332222210ull;    // th[16] = {0,1,2,2,2,2,2,3,3,3,3,3,3,3,3,4}
      int classIdx = (int)((TH >> (4 * act)) & 15);
      int hv1, hv0, d1, d0, dirHV, dirD;
      if (sV > sH) { hv1 = sV; hv0 = sH; dirHV = 1; } else { hv1 = sH; hv0 = sV; dirHV = 3; }
      if (sD0 > sD1) { d1 = sD0; d0 = sD1; dirD = 0; } else { d1 = sD1; d0 = sD0; dirD = 2; }
      int hvd1, hvd0, mainDir, secDir;
      if ((unsigned)d1 * (unsigned)hv0 > (unsigned)hv1 * (unsigned)d0) { hvd1 = d1; hvd0 = d0; mainDir = dirD; secDir = dirHV; }
      else { hvd1 = hv1; hvd0 = hv0; mainDir = dirHV; secDir = dirD; }
      int strength = 0;
      if (hvd1 > 2 * hvd0) strength = 1;
      if (hvd1 * 2 > 9 * hvd0) strength = 2;
      if (strength) classIdx += (((mainDir & 1) << 1) + strength) * 5;
      const unsigned TT = 0x31322010u;                         // transposeTable[8] = {0,1,0,2,2,3,1,3}
      const int tr = (TT >> (4 * (mainDir * 2 + (secDir >> 1)))) & 15;
      s_cls[b] = (uint16_t)(classIdx | (tr << 8));
    }
  }
  __syncthreads();

  // ---- 7x7 diamond (AdaptiveLoopFilter.cpp:1175): thread = row (tid>>3), 4 samples at x = (tid&7)*4 ----
  {
    const int ry = tid >> 3, rx = (tid & 7) * 4;
    if (ry >= bh || rx >= bw) return;
    const uint16_t k = s_cls[(ry >> 2) * 8 + (rx >> 2)];
    const int off = (k & 0xff) * 13 + (k >> 8) * 13 * 25 + cp.lumaSet * 4 * 25 * 13;
    const int16_t* f = P.lumaCoeff + off; const int16_t* c = P.lumaClip + off;
    int fc[12], cc[12];
#pragma unroll
    for (int i = 0; i < 12; i++) { fc[i] = __ldg(f + i); cc[i] = __ldg(c + i); }
    const int gy = by0 + ry;
    const int lim = alf_reach(gy & (vbH - 1), vbPos, 3);
    const int ly = ry + HALO;
    const int pmax = (1 << P.bitDepth) - 1;
    const int lx0 = rx + HALO;
    int out[4];
    bool wide = false;                                        // packed halves hold sums of two clipped differences of int8 weights
#pragma unroll
    for (int i = 0; i < 12; i++) wide |= fc[i] != (int)(int8_t)fc[i];
    if (!wide) {
      // w[3 + dy] = diamond row dy as aligned sample pairs from lx0 - 4 (lx0 is a multiple of 4); only the pairs the taps use are loaded
      uint32_t w[7][6];
#pragma unroll
      for (int dy = -3; dy <= 3; dy++) {
        const uint32_t* R = reinterpret_cast<const uint32_t*>(&t[ly + (dy < 0 ? -min(-dy, lim) : min(dy, lim))][0]) + (lx0 >> 1) - 2;
#pragma unroll
        for (int j = 0; j < 6; j++) w[dy + 3][j] = R[j];
      }
      int accLo[2] = {0, 0}, accHi[2] = {0, 0};
      const uint32_t ncur[2] = {__vneg2(w[3][2]), __vneg2(w[3][3])};
#pragma unroll
      for (int n = 0; n < 12; n++) {
        const int dy = ALF7[n].dy, dx = ALF7[n].dx;
        const uint32_t cl = (uint32_t)cc[n] * 0x10001u, cn = __vneg2(cl); const int kl = fc[n] & 0xff, kh = kl << 8;
#pragma unroll
        for (int q = 0; q < 2; q++) {                          // output samples lx0 + 2q, lx0 + 2q + 1
          const uint32_t d = __vmins2(__vmaxs2(__vadd2(alf_pair(w[3 + dy], 2 * q + dx), ncur[q]), cn), cl);
          const uint32_t e = __vmins2(__vmaxs2(__vadd2(alf_pair(w[3 - dy], 2 * q - dx), ncur[q]), cn), cl);
          const int de = (int)__vadd2(d, e);
          accLo[q] = __dp2a_lo(de, kl, accLo[q]); accHi[q] = __dp2a_lo(de, kh, accHi[q]);
        }
      }
#pragma unroll
      for (int q = 0; q < 2; q++) {
        const int c0 = (int)(int16_t)(w[3][2 + q] & 0xffff), c1 = (int)w[3][2 + q] >> 16;
        const int s0 = lim == 0 ? (accLo[q] + 512) >> 10 : (accLo[q] + 64) >> 7, s1 = lim == 0 ? (accHi[q] + 512) >> 10 : (accHi[q] + 64) >> 7;
        out[2 * q] = clip3(0, pmax, s0 + c0); out[2 * q + 1] = clip3(0, pmax, s1 + c1);
      }
    } else {
      // the 4 outputs share most taps: s[3 + dy][3 + j] = sample lx0 + j of diamond row dy, only the diamond's union loaded (46 samples instead of 4 x 25)
      int s[7][10];
#pragma unroll
      for (int dy = -3; dy <= 3; dy++) {
#pragma unroll
        for (int j = 0; j < 10; j++) s[dy + 3][j] = t[ly + (dy < 0 ? -min(-dy, lim) : min(dy, lim))][lx0 - 3 + j];
      }
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int cur = s[3][i + 3];
        int sum = 0;
#pragma unroll
        for (int n = 0; n < 12; n++) sum += fc[n] * clipd(cc[n], cur, s[3 + ALF7[n].dy][i + 3 + ALF7[n].dx], s[3 - ALF7[n].dy][i + 3 - ALF7[n].dx]);
        sum = lim == 0 ? (sum + 512) >> 10 : (sum + 64) >> 7;
        out[i] = clip3(0, pmax, sum + cur);
      }
    }
    *reinterpret_cast<uint2*>(P.dst[0] + (size_t)gy * stride + bx0 + rx) = pack4(out);
  }
}

// chroma 5x5 diamond + CC-ALF, 4:2:0. One thread per 4 chroma samples of one component; rows come through alf_window.
__global__ void __launch_bounds__(256) alf_chroma_kernel(const AlfParams P)
{
  const int c = 1 + blockIdx.z;
  const int pw = P.W >> 1, ph = P.H >> 1;
  const int x = (blockIdx.x * 32 + threadIdx.x) * 4, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= pw || y >= ph) return;
  const int l2cs = P.ctuLog2 - 1, cs = 1 << l2cs;
  const b200_alf_ctu cp = P.ctus[(y >> l2cs) * P.ctusW + (x >> l2cs)];
  // the component's plane and record fields by name: a runtime index would put the parameter block's arrays or the record on the stack
  const int enable = c == 1 ? cp.enable[1] : cp.enable[2], ccIdx = c == 1 ? cp.ccIdx[0] : cp.ccIdx[1];
  const int clipF = cp.enable[0] & ~1;
  const AlfView v = alf_view(c == 1 ? P.src[1] : P.src[2], c == 1 ? P.stride[1] : P.stride[2], pw, ph, l2cs, x, y, clipF, (enable & B200_ALF_PAD_WIDE) ? 2 : 0);
  const int pmax = (1 << P.bitDepth) - 1;
  const bool inner = x >= 4 && x + 8 <= pw && !clipF;
  int out[4];
  if (enable & 1) {
    const int alt = c == 1 ? cp.chromaAlt[0] : cp.chromaAlt[1];
    const int16_t* f = P.chromaCoeff + alt * 7; const int16_t* cl = P.chromaClip + alt * 7;
    int fc[6], cc[6];
#pragma unroll
    for (int i = 0; i < 6; i++) { fc[i] = __ldg(f + i); cc[i] = __ldg(cl + i); }
    const int lim = alf_reach(y & (cs - 1), cs - 2, 2), r1 = min(1, lim), r2 = min(2, lim);
    int s[5][8];                                              // s[2 + dy][2 + j] = sample x + j of diamond row dy
    alf_window<-2, 8>(v, x, y, inner, s[2]);
    alf_window<-1, 6>(v, x, y + r1, inner, s[3] + 1); alf_window<-1, 6>(v, x, y - r1, inner, s[1] + 1);
    alf_window<0, 4>(v, x, y + r2, inner, s[4] + 2);  alf_window<0, 4>(v, x, y - r2, inner, s[0] + 2);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int cur = s[2][i + 2];
      int sum = 0;
#pragma unroll
      for (int n = 0; n < 6; n++) sum += fc[n] * clipd(cc[n], cur, s[2 + ALF5[n].dy][i + 2 + ALF5[n].dx], s[2 - ALF5[n].dy][i + 2 - ALF5[n].dx]);
      sum = lim == 0 ? (sum + 512) >> 10 : (sum + 64) >> 7;
      out[i] = clip3(0, pmax, sum + cur);
    }
  } else {
    unpack4(*reinterpret_cast<const uint2*>(v.p + (size_t)y * v.stride + x), out);
  }
  if (ccIdx) {   // filterBlkCcAlf (AdaptiveLoopFilter.cpp:1348): 7-tap luma-difference filter on the PRE-ALF luma
    const int16_t* f = (c == 1 ? P.cc0 : P.cc1) + (ccIdx - 1) * 7;
    int fc[7];
#pragma unroll
    for (int i = 0; i < 7; i++) fc[i] = __ldg(f + i);
    const AlfView lv = alf_view(P.src[0], P.stride[0], P.W, P.H, P.ctuLog2, 2 * x, 2 * y, clipF, 0);
    const int ly = y << 1;
    int o1, o2, o3;
    ccalf_rows(ly & (P.ctuSize - 1), P.ctuSize - 4, o1, o2, o3);
    const int half = (1 << P.bitDepth) >> 1;
    // luma windows from 2x - 1 of rows ly, ly + o1 (9 samples); from 2x of rows ly + o2, ly + o3 (8 samples, the even ones used)
    int a[9], bb[9], up[8], dn[8];
    alf_window<-1, 9>(lv, 2 * x, ly, inner, a); alf_window<-1, 9>(lv, 2 * x, ly + o1, inner, bb);
    alf_window<0, 8>(lv, 2 * x, ly + o2, inner, up); alf_window<0, 8>(lv, 2 * x, ly + o3, inner, dn);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int cur = a[2 * i + 1];
      int sum = fc[0] * (up[2 * i] - cur) + fc[1] * (a[2 * i] - cur) + fc[2] * (a[2 * i + 2] - cur)
              + fc[3] * (bb[2 * i] - cur) + fc[4] * (bb[2 * i + 1] - cur) + fc[5] * (bb[2 * i + 2] - cur)
              + fc[6] * (dn[2 * i] - cur);
      sum = (sum + 64) >> 7;
      sum = clip3(0, pmax, sum + half) - half;
      out[i] = clip3(0, pmax, sum + out[i]);
    }
  }
  *reinterpret_cast<uint2*>((c == 1 ? P.dst[1] : P.dst[2]) + (size_t)y * v.stride + x) = pack4(out);
}

int launch_alf(const AlfLaunch& L, StreamSet& ss, KHook* hook)
{
  cudaStream_t s = ss.main;
  AlfParams P;
  for (int c = 0; c < 3; c++) { P.src[c] = L.src.p[c]; P.dst[c] = L.dst.p[c]; P.stride[c] = L.src.stride[c]; }
  P.W = L.geom.width; P.H = L.geom.height; P.bitDepth = L.geom.bitDepth; P.ctuSize = L.geom.ctuSize;
  P.ctuLog2 = ctu_log2(L.geom); P.ctusW = (P.W + P.ctuSize - 1) / P.ctuSize;
  P.ctus = L.ctus; P.lumaCoeff = L.lumaCoeff; P.lumaClip = L.lumaClip; P.chromaCoeff = L.chromaCoeff; P.chromaClip = L.chromaClip;
  P.cc0 = L.cc[0]; P.cc1 = L.cc[1];
  dim3 grdL((P.W + TB - 1) / TB, (P.H + TB - 1) / TB);
  if (L.geom.chromaFormat == 1) {                           // chroma + CC-ALF only read the SAO output: runs beside the luma kernel
    cudaStream_t sc = ss.pick(0);
    dim3 blk(32, 8), grd(((P.W >> 1) / 4 + 31) / 32, ((P.H >> 1) + 7) / 8, 2);
    hook_begin(hook, B200_KF_ALF_CHROMA, sc);
    alf_chroma_kernel<<<grd, blk, 0, sc>>>(P); hook_count(hook);
    B200_CUDA(cudaGetLastError());
    hook_end(hook, B200_KF_ALF_CHROMA, sc);
  }
  hook_begin(hook, B200_KF_ALF_LUMA, s);
  alf_luma_kernel<<<grdL, 256, 0, s>>>(P); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  hook_end(hook, B200_KF_ALF_LUMA, s);
  ss.join();
  return 0;
}

}  // namespace b200
