// k5_alf.cu — K5: adaptive loop filter. Luma: one CTA per 32x32 block (the reference's classification block): the block
// plus a 4-sample halo is staged in shared memory (coordinates clamped to the picture = prepareCTU's border extension),
// 4 threads per 4x4 block compute the Laplacian sums (warp-shuffle reduce), then every thread filters 4 samples with
// the 7x7 diamond, two output samples per 32-bit lane: packed 16-bit subtract / clamp (VIADD.16x2, VIMNMX.S16x2) and a
// 16x8-bit dot product per tap (IDP.2A); coefficients outside int8 (only +128 is legal) fall back to scalar arithmetic.  Chroma: one thread per 4 samples does the 5x5 diamond and adds CC-ALF from the pre-ALF luma.
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
  int vecOk;                      // luma stride is a multiple of 4 samples: rows can be copied 8 bytes at a time
  int vecOkC;                     // the same for all three planes (chroma kernel: chroma rows and the co-located luma rows)
  const b200_alf_ctu* ctus;
  const int16_t *lumaCoeff, *lumaClip, *chromaCoeff, *chromaClip, *cc0, *cc1;
};

__device__ __forceinline__ void cp_async8(void* smemDst, const void* gmemSrc)   // asynchronous 8-byte global -> shared copy (LDGSTS)
{
  const unsigned d = (unsigned)__cvta_generic_to_shared(smemDst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"(d), "l"(gmemSrc));
}

// CTUs whose neighbours may not be read (b200_alf_ctu::enable[0] bits, include/vvdec_b200.h): where a sample comes from.  (x0, y0)-(x1, y1): the CTU in the
// component's samples; pm: 0, or 2 for a chroma plane padded with the luma margin (B200_ALF_PAD_WIDE).
struct AlfExt { int x0, y0, x1, y1, W, H, f, pm; };
__device__ __forceinline__ void alf_map(const AlfExt& E, int& x, int& y)
{
  if ((E.f & B200_ALF_PAD_TL) && x < E.x0 + E.pm && y < E.y0 + E.pm) x = E.x0 + E.pm;             // raster-slice corners: the row's sample of the CTU's first / last column
  else if ((E.f & B200_ALF_PAD_BR) && x > E.x1 - E.pm && y > E.y1 - E.pm) x = E.x1 - E.pm;
  x = min(max(x, (E.f & B200_ALF_CLIP_LEFT) ? E.x0 : 0), (E.f & B200_ALF_CLIP_RIGHT) ? E.x1 : E.W - 1);
  y = min(max(y, (E.f & B200_ALF_CLIP_TOP) ? E.y0 : 0), (E.f & B200_ALF_CLIP_BOTTOM) ? E.y1 : E.H - 1);
}

__device__ __forceinline__ int clipd(int c, int ref, int a, int b) { return clip3(-c, c, a - ref) + clip3(-c, c, b - ref); }

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

  // ---- stage tile + halo, clamped ----
  const int clipF = cp.enable[0] & ~1;
  if (clipF) {                                              // a side of the CTU may not be read, or a corner is padded (filterCTU :763-848)
    AlfExt E; E.x0 = (bx0 >> P.ctuLog2) << P.ctuLog2; E.y0 = (by0 >> P.ctuLog2) << P.ctuLog2; E.x1 = min(E.x0 + P.ctuSize, P.W) - 1; E.y1 = min(E.y0 + P.ctuSize, P.H) - 1;
    E.W = P.W; E.H = P.H; E.f = clipF; E.pm = 0;
    for (int i = tid; i < TS * TS; i += 256) {
      const int ty = i / TS, tx = i - ty * TS;
      int gx = bx0 + tx - HALO, gy = by0 + ty - HALO;
      alf_map(E, gx, gy);
      t[ty][tx] = P.src[0][(size_t)gy * stride + gx];
    }
  } else if (P.vecOk && bx0 >= HALO && bx0 + TB + HALO <= P.W && by0 >= HALO && by0 + TB + HALO <= P.H) {
    const int16_t* s0 = P.src[0] + (size_t)(by0 - HALO) * stride + bx0 - HALO;      // interior tile: 40 rows x 10 8-byte words
    for (int i = tid; i < TS * (TS / 4); i += 256) {
      const int ty = i / (TS / 4), c = i - ty * (TS / 4);
      cp_async8(&t[ty][c * 4], reinterpret_cast<const uint2*>(s0 + (size_t)ty * stride) + c);
    }
    asm volatile("cp.async.wait_all;\n" ::: "memory");
  } else {
    for (int i = tid; i < TS * TS; i += 256) {
      const int ty = i / TS, tx = i - ty * TS;
      const int gx = min(max(bx0 + tx - HALO, 0), P.W - 1), gy = min(max(by0 + ty - HALO, 0), P.H - 1);
      t[ty][tx] = P.src[0][(size_t)gy * stride + gx];
    }
  }
  __syncthreads();

  const int vbH = P.ctuSize, vbPos = P.ctuSize - 4;

  // ---- classification (AdaptiveLoopFilter.cpp:969): thread = (4x4 block b, row pair r) ----
  {
    const int b = tid >> 2, r = tid & 3;
    const int bxi = b & 7, byi = b >> 3;
    const int y0 = by0 + byi * 4, x0l = bxi * 4;              // block origin: global y, tile-local x
    const bool aboveVb = (y0 & (vbH - 1)) == vbPos - 4, belowVb = (y0 & (vbH - 1)) == vbPos;
    int sV = 0, sH = 0, sD0 = 0, sD1 = 0;
    const bool skip = (aboveVb && r == 3) || (belowVb && r == 0);
    if (!skip) {
      const int gy = y0 - 2 + 2 * r;                          // first row of the pair (global)
      const int ly = byi * 4 - 2 + 2 * r + HALO;              // tile row
      int up = -1, dn2 = 2;
      if (gy > 0 && (gy & (vbH - 1)) == vbPos - 2) dn2 = 1;
      else if (gy > 0 && (gy & (vbH - 1)) == vbPos) up = 0;
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
      const int act = clip3(0, 15, ((sV + sH) * ((aboveVb || belowVb) ? 96 : 64)) >> shift);
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
    const int gy = by0 + ry, yVb = gy & (vbH - 1);
    int lim = 3;
    if (yVb < vbPos && yVb >= vbPos - 4) lim = vbPos - 1 - yVb;
    else if (yVb >= vbPos && yVb <= vbPos + 3) lim = yVb - vbPos;
    const bool nearVb = yVb == vbPos - 1 || yVb == vbPos;
    const int r1 = min(1, lim), r2 = min(2, lim), r3 = min(3, lim);
    const int ly = ry + HALO;
    const int pmax = (1 << P.bitDepth) - 1;
    const int lx0 = rx + HALO;
    int out[4];
    bool wide = P.bitDepth > 12;                              // packed halves hold sums of two clipped differences: 2 * 2^bd must fit 16 bit
#pragma unroll
    for (int i = 0; i < 12; i++) wide |= fc[i] != (int)(int8_t)fc[i];
    if (!wide) {
      // rows as aligned sample pairs (lx0 is a multiple of 4); odd offsets are built with one byte-permute from two neighbours
      const uint32_t* R0 = reinterpret_cast<const uint32_t*>(&t[ly][0]) + (lx0 >> 1);
      const uint32_t* P1 = reinterpret_cast<const uint32_t*>(&t[ly + r1][0]) + (lx0 >> 1); const uint32_t* M1 = reinterpret_cast<const uint32_t*>(&t[ly - r1][0]) + (lx0 >> 1);
      const uint32_t* P2 = reinterpret_cast<const uint32_t*>(&t[ly + r2][0]) + (lx0 >> 1); const uint32_t* M2 = reinterpret_cast<const uint32_t*>(&t[ly - r2][0]) + (lx0 >> 1);
      const uint32_t* P3 = reinterpret_cast<const uint32_t*>(&t[ly + r3][0]) + (lx0 >> 1); const uint32_t* M3 = reinterpret_cast<const uint32_t*>(&t[ly - r3][0]) + (lx0 >> 1);
      uint32_t r0w[6], p1w[4], m1w[4], p2w[4], m2w[4], p3w[2], m3w[2];
#pragma unroll
      for (int k = 0; k < 6; k++) r0w[k] = R0[k - 2];                                  // samples lx0-4 .. lx0+7
#pragma unroll
      for (int k = 0; k < 4; k++) { p1w[k] = P1[k - 1]; m1w[k] = M1[k - 1]; p2w[k] = P2[k - 1]; m2w[k] = M2[k - 1]; }   // lx0-2 .. lx0+5
#pragma unroll
      for (int k = 0; k < 2; k++) { p3w[k] = P3[k]; m3w[k] = M3[k]; }
      uint32_t r0s[5], p1s[3], m1s[3], p2s[3], m2s[3];                                 // pairs starting at odd offsets
#pragma unroll
      for (int k = 0; k < 5; k++) r0s[k] = __byte_perm(r0w[k], r0w[k + 1], 0x5432);   // offsets -3,-1,1,3,5
#pragma unroll
      for (int k = 0; k < 3; k++) {                                                    // offsets -1,1,3
        p1s[k] = __byte_perm(p1w[k], p1w[k + 1], 0x5432); m1s[k] = __byte_perm(m1w[k], m1w[k + 1], 0x5432);
        p2s[k] = __byte_perm(p2w[k], p2w[k + 1], 0x5432); m2s[k] = __byte_perm(m2w[k], m2w[k + 1], 0x5432);
      }
      int accLo[2] = {0, 0}, accHi[2] = {0, 0};
      uint32_t ncur[2] = {__vneg2(r0w[2]), __vneg2(r0w[3])};
      // pair of samples at offset j (relative to lx0) of each row, j compile-time
#define R0P(j) (((j) & 1) ? r0s[((j) + 3) >> 1] : r0w[((j) + 4) >> 1])
#define P1P(j) (((j) & 1) ? p1s[((j) + 1) >> 1] : p1w[((j) + 2) >> 1])
#define M1P(j) (((j) & 1) ? m1s[((j) + 1) >> 1] : m1w[((j) + 2) >> 1])
#define P2P(j) (((j) & 1) ? p2s[((j) + 1) >> 1] : p2w[((j) + 2) >> 1])
#define M2P(j) (((j) & 1) ? m2s[((j) + 1) >> 1] : m2w[((j) + 2) >> 1])
#define ALF_TAP(n, A0, B0, A1, B1) { \
        const uint32_t cp = (uint32_t)cc[n] * 0x10001u, cn = __vneg2(cp); const int kl = fc[n] & 0xff, kh = kl << 8; \
        uint32_t d0 = __vmins2(__vmaxs2(__vadd2(A0, ncur[0]), cn), cp), e0 = __vmins2(__vmaxs2(__vadd2(B0, ncur[0]), cn), cp); \
        uint32_t d1 = __vmins2(__vmaxs2(__vadd2(A1, ncur[1]), cn), cp), e1 = __vmins2(__vmaxs2(__vadd2(B1, ncur[1]), cn), cp); \
        d0 = __vadd2(d0, e0); d1 = __vadd2(d1, e1); \
        accLo[0] = __dp2a_lo((int)d0, kl, accLo[0]); accHi[0] = __dp2a_lo((int)d0, kh, accHi[0]); \
        accLo[1] = __dp2a_lo((int)d1, kl, accLo[1]); accHi[1] = __dp2a_lo((int)d1, kh, accHi[1]); }
      ALF_TAP(0,  p3w[0],  m3w[0],  p3w[1],  m3w[1])
      ALF_TAP(1,  P2P(1),  M2P(-1), P2P(3),  M2P(1))
      ALF_TAP(2,  P2P(0),  M2P(0),  P2P(2),  M2P(2))
      ALF_TAP(3,  P2P(-1), M2P(1),  P2P(1),  M2P(3))
      ALF_TAP(4,  P1P(2),  M1P(-2), P1P(4),  M1P(0))
      ALF_TAP(5,  P1P(1),  M1P(-1), P1P(3),  M1P(1))
      ALF_TAP(6,  P1P(0),  M1P(0),  P1P(2),  M1P(2))
      ALF_TAP(7,  P1P(-1), M1P(1),  P1P(1),  M1P(3))
      ALF_TAP(8,  P1P(-2), M1P(2),  P1P(0),  M1P(4))
      ALF_TAP(9,  R0P(3),  R0P(-3), R0P(5),  R0P(-1))
      ALF_TAP(10, R0P(2),  R0P(-2), R0P(4),  R0P(0))
      ALF_TAP(11, R0P(1),  R0P(-1), R0P(3),  R0P(1))
#undef ALF_TAP
#undef R0P
#undef P1P
#undef M1P
#undef P2P
#undef M2P
#pragma unroll
      for (int q = 0; q < 2; q++) {
        const int c0 = (int)(int16_t)(r0w[2 + q] & 0xffff), c1 = (int)r0w[2 + q] >> 16;
        const int s0 = nearVb ? (accLo[q] + 512) >> 10 : (accLo[q] + 64) >> 7, s1 = nearVb ? (accHi[q] + 512) >> 10 : (accHi[q] + 64) >> 7;
        out[2 * q] = clip3(0, pmax, s0 + c0); out[2 * q + 1] = clip3(0, pmax, s1 + c1);
      }
    } else {
    // the 4 outputs share most taps: fetch the diamond's union once (46 samples instead of 4 x 25)
    int r0[10], p1[8], m1[8], p2[6], m2[6], p3[4], m3[4];
#pragma unroll
    for (int k = 0; k < 10; k++) r0[k] = t[ly][lx0 - 3 + k];
#pragma unroll
    for (int k = 0; k < 8; k++) { p1[k] = t[ly + r1][lx0 - 2 + k]; m1[k] = t[ly - r1][lx0 - 2 + k]; }
#pragma unroll
    for (int k = 0; k < 6; k++) { p2[k] = t[ly + r2][lx0 - 1 + k]; m2[k] = t[ly - r2][lx0 - 1 + k]; }
#pragma unroll
    for (int k = 0; k < 4; k++) { p3[k] = t[ly + r3][lx0 + k]; m3[k] = t[ly - r3][lx0 + k]; }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int cur = r0[i + 3];
      int sum = 0;
      sum += fc[0]  * clipd(cc[0],  cur, p3[i],     m3[i]);
      sum += fc[1]  * clipd(cc[1],  cur, p2[i + 2], m2[i]);
      sum += fc[2]  * clipd(cc[2],  cur, p2[i + 1], m2[i + 1]);
      sum += fc[3]  * clipd(cc[3],  cur, p2[i],     m2[i + 2]);
      sum += fc[4]  * clipd(cc[4],  cur, p1[i + 4], m1[i]);
      sum += fc[5]  * clipd(cc[5],  cur, p1[i + 3], m1[i + 1]);
      sum += fc[6]  * clipd(cc[6],  cur, p1[i + 2], m1[i + 2]);
      sum += fc[7]  * clipd(cc[7],  cur, p1[i + 1], m1[i + 3]);
      sum += fc[8]  * clipd(cc[8],  cur, p1[i],     m1[i + 4]);
      sum += fc[9]  * clipd(cc[9],  cur, r0[i + 6], r0[i]);
      sum += fc[10] * clipd(cc[10], cur, r0[i + 5], r0[i + 1]);
      sum += fc[11] * clipd(cc[11], cur, r0[i + 4], r0[i + 2]);
      sum = nearVb ? (sum + 512) >> 10 : (sum + 64) >> 7;
      out[i] = clip3(0, pmax, sum + cur);
    }
    }
    uint2 o;
    o.x = (unsigned)(out[0] & 0xffff) | ((unsigned)out[1] << 16);
    o.y = (unsigned)(out[2] & 0xffff) | ((unsigned)out[3] << 16);
    *reinterpret_cast<uint2*>(P.dst[0] + (size_t)gy * stride + bx0 + rx) = o;
  }
}

// chroma 5x5 diamond + CC-ALF, 4:2:0. One thread per 4 chroma samples of one component.  Threads away from the left / right picture
// edge fetch their rows as 8- / 16-byte vectors (row indices are clamped, which is the reference's border extension); edge threads
// read sample by sample with clamped coordinates.
__device__ __forceinline__ void unpack4(const uint2 u, int* d) { d[0] = (int)(int16_t)(u.x & 0xffff); d[1] = (int)u.x >> 16; d[2] = (int)(int16_t)(u.y & 0xffff); d[3] = (int)u.y >> 16; }

__global__ void __launch_bounds__(256) alf_chroma_kernel(const AlfParams P)
{
  const int c = 1 + blockIdx.z;
  const int pw = P.W >> 1, ph = P.H >> 1;
  const int x = (blockIdx.x * 32 + threadIdx.x) * 4, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= pw || y >= ph) return;
  const int l2cs = P.ctuLog2 - 1, cs = 1 << l2cs;
  const b200_alf_ctu cp = P.ctus[(y >> l2cs) * P.ctusW + (x >> l2cs)];
  const int stride = P.stride[c];
  const int16_t* s = P.src[c];
  const int pmax = (1 << P.bitDepth) - 1;
  const int clipF = cp.enable[0] & ~1;
  const bool inner = P.vecOkC && x >= 4 && x + 8 <= pw && !clipF;
  int out[4];
  AlfExt E; E.x0 = (x >> l2cs) << l2cs; E.y0 = (y >> l2cs) << l2cs; E.x1 = min(E.x0 + cs, pw) - 1; E.y1 = min(E.y0 + cs, ph) - 1; E.W = pw; E.H = ph; E.f = clipF;
  E.pm = (cp.enable[c] & B200_ALF_PAD_WIDE) ? 2 : 0;
  auto rowp = [&](int yy) { return s + (size_t)min(max(yy, 0), ph - 1) * stride; };
  auto at = [&](int xx, int yy) { if (clipF) { alf_map(E, xx, yy); return (int)s[(size_t)yy * stride + xx]; } return (int)rowp(yy)[min(max(xx, 0), pw - 1)]; };
  if (cp.enable[c] & 1) {
    const int16_t* f = P.chromaCoeff + cp.chromaAlt[c - 1] * 7; const int16_t* cl = P.chromaClip + cp.chromaAlt[c - 1] * 7;
    int fc[6], cc[6];
#pragma unroll
    for (int i = 0; i < 6; i++) { fc[i] = __ldg(f + i); cc[i] = __ldg(cl + i); }
    const int vbH = cs, vbPos = cs - 2, yVb = y & (vbH - 1);
    int lim = 2;
    if (yVb < vbPos && yVb >= vbPos - 2) lim = vbPos - 1 - yVb;
    else if (yVb >= vbPos && yVb <= vbPos + 1) lim = yVb - vbPos;
    const bool nearVb = yVb == vbPos - 1 || yVb == vbPos;
    const int r1 = min(1, lim), r2 = min(2, lim);
    // rows as windows: r0[k] = sample x-2+k (8), p1/m1[k] = sample x-1+k of rows y+-r1 (6), p2/m2[k] = sample x+k of rows y+-r2 (4)
    int r0[8], p1[6], m1[6], p2[4], m2[4];
    if (inner) {
      int t[4];
      const int16_t* q = rowp(y) + x;
      unpack4(__ldg(reinterpret_cast<const uint2*>(q - 4)), t); r0[0] = t[2]; r0[1] = t[3];
      unpack4(__ldg(reinterpret_cast<const uint2*>(q)), r0 + 2);
      unpack4(__ldg(reinterpret_cast<const uint2*>(q + 4)), t); r0[6] = t[0]; r0[7] = t[1];
      q = rowp(y + r1) + x; p1[0] = q[-1]; unpack4(__ldg(reinterpret_cast<const uint2*>(q)), p1 + 1); p1[5] = q[4];
      q = rowp(y - r1) + x; m1[0] = q[-1]; unpack4(__ldg(reinterpret_cast<const uint2*>(q)), m1 + 1); m1[5] = q[4];
      unpack4(__ldg(reinterpret_cast<const uint2*>(rowp(y + r2) + x)), p2);
      unpack4(__ldg(reinterpret_cast<const uint2*>(rowp(y - r2) + x)), m2);
    } else {
#pragma unroll
      for (int k = 0; k < 8; k++) r0[k] = at(x - 2 + k, y);
#pragma unroll
      for (int k = 0; k < 6; k++) { p1[k] = at(x - 1 + k, y + r1); m1[k] = at(x - 1 + k, y - r1); }
#pragma unroll
      for (int k = 0; k < 4; k++) { p2[k] = at(x + k, y + r2); m2[k] = at(x + k, y - r2); }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int cur = r0[i + 2];
      int sum = 0;
      sum += fc[0] * clipd(cc[0], cur, p2[i],     m2[i]);
      sum += fc[1] * clipd(cc[1], cur, p1[i + 2], m1[i]);
      sum += fc[2] * clipd(cc[2], cur, p1[i + 1], m1[i + 1]);
      sum += fc[3] * clipd(cc[3], cur, p1[i],     m1[i + 2]);
      sum += fc[4] * clipd(cc[4], cur, r0[i + 4], r0[i]);
      sum += fc[5] * clipd(cc[5], cur, r0[i + 3], r0[i + 1]);
      sum = nearVb ? (sum + 512) >> 10 : (sum + 64) >> 7;
      out[i] = clip3(0, pmax, sum + cur);
    }
  } else {
    unpack4(*reinterpret_cast<const uint2*>(s + (size_t)y * stride + x), out);
  }
  const int ccIdx = cp.ccIdx[c - 1];
  if (ccIdx) {   // filterBlkCcAlf (AdaptiveLoopFilter.cpp:1348): 7-tap luma-difference filter on the PRE-ALF luma
    const int16_t* f = (c == 1 ? P.cc0 : P.cc1) + (ccIdx - 1) * 7;
    int fc[7];
#pragma unroll
    for (int i = 0; i < 7; i++) fc[i] = __ldg(f + i);
    const int16_t* L = P.src[0]; const int ls = P.stride[0];
    const int ly = y << 1, pos = ly & (P.ctuSize - 1), vbPos = P.ctuSize - 4;
    int o1 = 1, o2 = -1, o3 = 2;
    if (pos == vbPos - 2 || pos == vbPos + 1) o3 = 1;
    else if (pos == vbPos - 1 || pos == vbPos) o1 = o2 = o3 = 0;
    AlfExt EL; EL.x0 = E.x0 << 1; EL.y0 = E.y0 << 1; EL.x1 = min(EL.x0 + P.ctuSize, P.W) - 1; EL.y1 = min(EL.y0 + P.ctuSize, P.H) - 1; EL.W = P.W; EL.H = P.H; EL.f = clipF; EL.pm = 0;
    auto lrow = [&](int yy) { return L + (size_t)min(max(yy, 0), P.H - 1) * ls; };
    auto lat = [&](int xx, int yy) { if (clipF) { alf_map(EL, xx, yy); return (int)L[(size_t)yy * ls + xx]; } return (int)lrow(yy)[min(max(xx, 0), P.W - 1)]; };
    const int half = (1 << P.bitDepth) >> 1;
    // luma windows: a[k], b[k] = luma sample 2x-1+k of rows ly, ly+o1 (9); up[i], dn[i] = luma sample 2(x+i) of rows ly+o2, ly+o3
    int a[9], bb[9], up[4], dn[4];
    if (inner) {
      int t[4];
      const int16_t* q = lrow(ly) + 2 * x;
      a[0] = q[-1]; unpack4(__ldg(reinterpret_cast<const uint2*>(q)), a + 1); unpack4(__ldg(reinterpret_cast<const uint2*>(q + 4)), a + 5);
      q = lrow(ly + o1) + 2 * x;
      bb[0] = q[-1]; unpack4(__ldg(reinterpret_cast<const uint2*>(q)), bb + 1); unpack4(__ldg(reinterpret_cast<const uint2*>(q + 4)), bb + 5);
      q = lrow(ly + o2) + 2 * x;
      unpack4(__ldg(reinterpret_cast<const uint2*>(q)), t); up[0] = t[0]; up[1] = t[2]; unpack4(__ldg(reinterpret_cast<const uint2*>(q + 4)), t); up[2] = t[0]; up[3] = t[2];
      q = lrow(ly + o3) + 2 * x;
      unpack4(__ldg(reinterpret_cast<const uint2*>(q)), t); dn[0] = t[0]; dn[1] = t[2]; unpack4(__ldg(reinterpret_cast<const uint2*>(q + 4)), t); dn[2] = t[0]; dn[3] = t[2];
    } else {
#pragma unroll
      for (int k = 0; k < 9; k++) { a[k] = lat(2 * x - 1 + k, ly); bb[k] = lat(2 * x - 1 + k, ly + o1); }
#pragma unroll
      for (int i = 0; i < 4; i++) { up[i] = lat(2 * (x + i), ly + o2); dn[i] = lat(2 * (x + i), ly + o3); }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int cur = a[2 * i + 1];
      int sum = fc[0] * (up[i] - cur) + fc[1] * (a[2 * i] - cur) + fc[2] * (a[2 * i + 2] - cur)
              + fc[3] * (bb[2 * i] - cur) + fc[4] * (bb[2 * i + 1] - cur) + fc[5] * (bb[2 * i + 2] - cur)
              + fc[6] * (dn[i] - cur);
      sum = (sum + 64) >> 7;
      sum = clip3(0, pmax, sum + half) - half;
      out[i] = clip3(0, pmax, sum + out[i]);
    }
  }
  uint2 o;
  o.x = (unsigned)(out[0] & 0xffff) | ((unsigned)out[1] << 16);
  o.y = (unsigned)(out[2] & 0xffff) | ((unsigned)out[3] << 16);
  *reinterpret_cast<uint2*>(P.dst[c] + (size_t)y * stride + x) = o;
}

int launch_alf(const AlfLaunch& L, StreamSet& ss, KHook* hook)
{
  cudaStream_t s = ss.main;
  AlfParams P;
  for (int c = 0; c < 3; c++) { P.src[c] = L.src.p[c]; P.dst[c] = L.dst.p[c]; P.stride[c] = L.src.stride[c]; }
  P.W = L.geom.width; P.H = L.geom.height; P.bitDepth = L.geom.bitDepth; P.ctuSize = L.geom.ctuSize;
  P.ctuLog2 = P.ctuSize == 128 ? 7 : P.ctuSize == 64 ? 6 : 5; P.ctusW = (P.W + P.ctuSize - 1) / P.ctuSize;
  P.ctus = L.ctus; P.lumaCoeff = L.lumaCoeff; P.lumaClip = L.lumaClip; P.chromaCoeff = L.chromaCoeff; P.chromaClip = L.chromaClip;
  P.cc0 = L.cc[0]; P.cc1 = L.cc[1];
  P.vecOk = (P.stride[0] & 3) == 0 && (reinterpret_cast<uintptr_t>(P.src[0]) & 7) == 0;
  P.vecOkC = P.vecOk && (P.stride[1] & 3) == 0 && (P.stride[2] & 3) == 0 && (reinterpret_cast<uintptr_t>(P.src[1]) & 7) == 0 && (reinterpret_cast<uintptr_t>(P.src[2]) & 7) == 0;
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
