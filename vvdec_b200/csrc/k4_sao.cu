// k4_sao.cu — K4: sample adaptive offset, src (deblocked) -> dst, one thread per 4 consecutive samples.
//
// Replaces (reference, source/Lib/CommonLib/SampleAdaptiveOffset.cpp): offsetBlock_core :64-349, SAOProcessCTU :522,
// offsetCTU :661, isProcessDisabled :817.  The CPU version walks lines with sign caches; per sample it is
//   EO: dst = clip(c + offset[2 + sgn(c-n0) + sgn(c-n1)]) if both neighbours along the class direction lie inside the
//       CTU or in an available neighbouring CTU and the sample is not adjacent to a virtual boundary; else dst = c
//   BO: dst = clip(c + offset[c >> (bd-5)])
// which is what each thread evaluates.  HBM traffic: S*2 B read (neighbour rows hit L1/L2) + S*2 B written + 24 B/CTU.
#include "common.cuh"

namespace b200 {

struct SaoParams {
  const int16_t* src[3]; int16_t* dst[3]; int stride[3];
  int W, H, bitDepth, ctuSize, ctuLog2, ctusW, chroma;
  const b200_sao_ctu* ctus;
  b200_vb vb;
};

__device__ __forceinline__ int sgn(int v) { return (v > 0) - (v < 0); }

__global__ void __launch_bounds__(256) sao_kernel(const SaoParams P)
{
  const int c = blockIdx.z;
  const int sh = c ? 1 : 0;
  const int pw = P.W >> sh, ph = P.H >> sh;
  const int x = (blockIdx.x * 32 + threadIdx.x) * 4, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= pw || y >= ph) return;
  const int stride = c == 0 ? P.stride[0] : c == 1 ? P.stride[1] : P.stride[2];
  const int16_t* s = c == 0 ? P.src[0] : c == 1 ? P.src[1] : P.src[2];
  const int l2cs = P.ctuLog2 - sh, cs = 1 << l2cs;            // CTU size in this plane
  const int cxi = x >> l2cs, cyi = y >> l2cs;
  const uint8_t* rec = reinterpret_cast<const uint8_t*>(P.ctus + cyi * P.ctusW + cxi);   // 24-byte record, one L1 line for the whole warp
  const int type = __ldg(rec + c);
  uint2* dptr = reinterpret_cast<uint2*>((c == 0 ? P.dst[0] : c == 1 ? P.dst[1] : P.dst[2]) + (size_t)y * stride + x);
  const uint2 ctr = *reinterpret_cast<const uint2*>(s + (size_t)y * stride + x);
  if (type == B200_SAO_OFF) { *dptr = ctr; return; }
  // the component's five offsets as bytes 0..4 of a word pair: one byte-permute selects offset[k]
  const uint8_t* ob = rec + 6 + c * 5;
  const uint32_t offLo = __ldg(ob) | (__ldg(ob + 1) << 8) | (__ldg(ob + 2) << 16) | (__ldg(ob + 3) << 24), offHi = __ldg(ob + 4);
  auto offset_of = [&](int k) -> int { return (int)(int8_t)__byte_perm(offLo, offHi, k); };
  int v[4];
  unpack4(ctr, v);
  int r[4] = { v[0], v[1], v[2], v[3] };
  const int pmax = (1 << P.bitDepth) - 1;
  if (type == B200_SAO_BO) {
    const int shiftBits = P.bitDepth - 5, band = __ldg(rec + 3 + c);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int k = ((v[i] >> shiftBits) - band) & 31;
      if (k < 4) r[i] = clip3(0, pmax, v[i] + offset_of(k));
    }
  } else {
    // neighbour offsets of the class: EO_0 (-1,0)/(+1,0); EO_90 (0,-1)/(0,+1); EO_135 (-1,-1)/(+1,+1); EO_45 (+1,-1)/(-1,+1)
    const int dx = type == B200_SAO_EO_90 ? 0 : (type == B200_SAO_EO_45 ? -1 : 1);
    const int dy = type == B200_SAO_EO_0 ? 0 : 1;
    const int x0c = cxi << l2cs, y0c = cyi << l2cs;
    const int w = min(cs, pw - x0c), h = min(cs, ph - y0c);
    const int lx = x - x0c, ly = y - y0c;
    // neighbour samples of the 4 outputs, fetched as two 8-byte vectors + at most two scalars (rows / columns clamped: clamped
    // values are only ever used by samples that the availability test rejects)
    int na[4], nb[4];
    {
      const int16_t* rowA = s + (size_t)max(y - dy, 0) * stride;
      const int16_t* rowB = s + (size_t)min(y + dy, ph - 1) * stride;
      const int xl = max(x - 1, 0), xr = min(x + 4, pw - 1);
      if (dy == 0) {
        const int l = rowA[xl], r4 = rowA[xr];
        na[0] = l; na[1] = v[0]; na[2] = v[1]; na[3] = v[2]; nb[0] = v[1]; nb[1] = v[2]; nb[2] = v[3]; nb[3] = r4;
      } else {
        const uint2 ua = *reinterpret_cast<const uint2*>(rowA + x), ub = *reinterpret_cast<const uint2*>(rowB + x);
        int A[4], B[4];
        unpack4(ua, A); unpack4(ub, B);
        if (dx == 0)      { na[0] = A[0]; na[1] = A[1]; na[2] = A[2]; na[3] = A[3]; nb[0] = B[0]; nb[1] = B[1]; nb[2] = B[2]; nb[3] = B[3]; }
        else if (dx == 1) { na[0] = rowA[xl]; na[1] = A[0]; na[2] = A[1]; na[3] = A[2]; nb[0] = B[1]; nb[1] = B[2]; nb[2] = B[3]; nb[3] = rowB[xr]; }
        else              { na[0] = A[1]; na[1] = A[2]; na[2] = A[3]; na[3] = rowA[xr]; nb[0] = rowB[xl]; nb[1] = B[0]; nb[2] = B[1]; nb[3] = B[2]; }
      }
    }
    // which of the 4 samples may be filtered (bit i): both neighbours must lie in the CTU or in an available neighbouring CTU.
    // Neighbour A = (-dx,-dy) is above (dy = 1) or in the row; only sample 0 / 3 of a thread on the CTU's left / right column can
    // leave the CTU sideways.
    unsigned okMask = 0xf;
    if (ly == 0 || ly == h - 1 || lx == 0 || lx + 4 >= w) {
      const unsigned avail = __ldg(rec + 21);
      const bool up = dy && ly == 0, dn = dy && ly == h - 1;
      const unsigned midA = up ? B200_AVAIL_A : 0, leftA = up ? B200_AVAIL_AL : B200_AVAIL_L, rightA = up ? B200_AVAIL_AR : B200_AVAIL_R;
      const unsigned midB = dn ? B200_AVAIL_B : 0, leftB = dn ? B200_AVAIL_BL : B200_AVAIL_L, rightB = dn ? B200_AVAIL_BR : B200_AVAIL_R;
      unsigned a0 = midA, a3 = midA, b0 = midB, b3 = midB;   // requirements of neighbour A / B for sample 0 and sample 3 (1 and 2 stay inside)
      if (dx == 1)  { if (lx == 0) a0 = leftA;  if (lx + 4 == w) b3 = rightB; }   // A looks left, B looks right
      if (dx == -1) { if (lx + 4 == w) a3 = rightA; if (lx == 0) b0 = leftB; }    // A looks right, B looks left
      const unsigned need0 = a0 | b0, need3 = a3 | b3, needM = midA | midB;
      if ((need0 & avail) != need0) okMask &= ~1u;
      if ((needM & avail) != needM) okMask &= ~6u;
      if ((need3 & avail) != need3) okMask &= ~8u;
    }
    if (P.vb.numVer | P.vb.numHor) {                        // picture-uniform: virtual boundaries (samples next to one are not filtered)
      const int nV = type == B200_SAO_EO_90 ? 0 : P.vb.numVer, nH = type == B200_SAO_EO_0 ? 0 : P.vb.numHor;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int gx = x + i;
#pragma unroll
        for (int k = 0; k < 3; k++) { const int p = P.vb.posX[k] >> sh; if (k < nV && (gx == p || gx == p - 1)) okMask &= ~(1u << i); }
#pragma unroll
        for (int k = 0; k < 3; k++) { const int p = P.vb.posY[k] >> sh; if (k < nH && (y == p || y == p - 1)) okMask &= ~(1u << i); }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int e = sgn(v[i] - na[i]) + sgn(v[i] - nb[i]);
      if (okMask & (1u << i)) r[i] = clip3(0, pmax, v[i] + offset_of(e + 2));
    }
  }
  *dptr = pack4(r);
}

int launch_sao(const SaoLaunch& L, cudaStream_t s, KHook* hook)
{
  SaoParams P;
  for (int c = 0; c < 3; c++) { P.src[c] = L.src.p[c]; P.dst[c] = L.dst.p[c]; P.stride[c] = L.src.stride[c]; }
  P.W = L.geom.width; P.H = L.geom.height; P.bitDepth = L.geom.bitDepth; P.ctuSize = L.geom.ctuSize;
  P.ctuLog2 = ctu_log2(L.geom);
  P.ctusW = (P.W + P.ctuSize - 1) / P.ctuSize; P.chroma = L.geom.chromaFormat == 1;
  P.ctus = L.ctus; P.vb = L.vb;
  dim3 blk(32, 8), grd((P.W / 4 + 31) / 32, (P.H + 7) / 8, P.chroma ? 3 : 1);
  hook_begin(hook, B200_KF_SAO, s);
  sao_kernel<<<grd, blk, 0, s>>>(P); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  hook_end(hook, B200_KF_SAO, s);
  return 0;
}

}  // namespace b200
