// film_grain.cu — film grain synthesis on the output frame (SURVEY 8f-3), the per-sample ("hardware") half of the reference's VFGS model.
// Replaces (reference, source/Lib/FilmGrain/): FilmGrainImpl::add_grain_block / make_grain_pattern / scale_and_output
// (FilmGrainImpl.cpp:129,:198,:247; SIMD: FilmGrainImpl_X86_SIMD.h:54,:392) and the line walk FilmGrain::add_grain_line (FilmGrain.cpp:836)
// that VVDecImpl::xAddGrain (vvdecimpl.cpp:898) runs in 16-line tasks.
//
// The reference streams each line through a two-block pipeline (grain of block b is smoothed against block b+1, then scaled and written
// when b+1 arrives).  Here the grain is a pure function G(x, y) of the sample position: block seed -> offsets/sign -> pattern sample chosen
// by the sample's intensity (+ the vertical blend with the block row above on the first two lines of a block row); the smoothing across a
// 16-sample block border is the 3-tap stencil (G(x-1) + 3 G(x) + G(x+1) + 2) >> 2 on the raw values of the two samples next to it.  One
// thread per sample; the 1/8 of the threads that sit at a border evaluate G three times.
// Scale LUT entries are unsigned as in the C model (FilmGrainImpl.cpp:282); the x86 SIMD class sign-extends them at 10 bit (DESIGN.md 4).
#include "common.cuh"

namespace b200 {

__device__ __forceinline__ uint32_t fg_prng(uint32_t x) { const uint32_t s = ((x << 30) ^ (x << 2)) & 0x80000000u; return s | (x >> 1); }

// block seeds: one prng step per 16-sample block along a line of blocks (add_grain_line :864), one thread per block row
__global__ void fg_seed_kernel(const uint32_t* __restrict__ lineSeeds, int nbx, int nby, uint32_t* __restrict__ seeds)
{
  const int by = blockIdx.x * blockDim.x + threadIdx.x;
  if (by >= nby) return;
  uint32_t r = lineSeeds[by];
  for (int bx = 0; bx < nbx; bx++) { seeds[by * nbx + bx] = r; r = fg_prng(r); }
}

struct FgParams {
  const int16_t* src[3]; int16_t* dst[3]; int srcStride[3], dstStride[3];
  int W, H, bs, scaleShift, nbx; uint8_t present[3];
  const int8_t* pattern; const uint8_t *sLUT, *pLUT; const uint32_t* seeds;
};

// offsets and sign of a block from its seed (get_offset_y/u/v :85-127); sub = chroma subsampling (2) or 1
template <int C> __device__ __forceinline__ void fg_offsets(uint32_t v, int sub, int& s, int& ox, int& oy)
{
  uint32_t bx, by;
  if (C == 0)      { s = (v >> 31) & 1; bx = v & 0x3ff; by = (v >> 14) & 0x3ff; }
  else if (C == 1) { s = (v >> 2) & 1;  bx = (v >> 10) & 0x3ff; by = ((v >> 24) & 0xff) | ((v << 8) & 0x300); }
  else             { s = (v >> 15) & 1; bx = (v >> 20) & 0x3ff; by = (v >> 4) & 0x3ff; }
  ox = (int)((bx * 13) >> 10) * (4 / sub); oy = (int)((by * 12) >> 10) * (4 / sub);
}

template <int C> __device__ __forceinline__ int fg_grain(const FgParams& P, const uint8_t* __restrict__ plut, int xs, int ys)
{
  constexpr int SUB = C ? 2 : 1, BW = 16 / SUB;
  const int y = ys * SUB, bx = xs / BW, i = xs - bx * BW, by = y >> 4, j = y & 15;
  int s, ox, oy;
  fg_offsets<C>(__ldg(P.seeds + by * P.nbx + bx), SUB, s, ox, oy);
  oy += j / SUB;
  const int intensity = (reinterpret_cast<const uint16_t*>(P.src[C])[(size_t)ys * P.srcStride[C] + xs] >> P.bs) & 0xff;
  const int8_t* pat = P.pattern + ((C ? 8 : 0) + (plut[intensity] >> 4)) * 4096;
  int g = __ldg(pat + oy * 64 + ox + i); if (s) g = -g;
  if (y > 15 && j < 2) {                                   // first two lines of a block row: blend with the pattern of the block above (:150-163)
    const int oc1 = j ? 24 : (SUB > 1 ? 20 : 12), oc2 = j ? 12 : (SUB > 1 ? 20 : 24);
    int sU, oxU, oyU;
    fg_offsets<C>(__ldg(P.seeds + (by - 1) * P.nbx + bx), SUB, sU, oxU, oyU);
    oyU += (16 + j) / SUB;
    int u = __ldg(pat + oyU * 64 + oxU + i); if (sU) u = -u;
    g = (g * oc1 + u * oc2 + 16) >> 5;
  }
  return g;
}

template <int C> __global__ void __launch_bounds__(256) fg_kernel(const FgParams P)
{
  constexpr int SUB = C ? 2 : 1, BW = 16 / SUB;
  __shared__ uint8_t lut[512];                             // pLUT[C], sLUT[C]
  for (int k = threadIdx.x; k < 512; k += 256) lut[k] = k < 256 ? P.pLUT[C * 256 + k] : P.sLUT[C * 256 + k - 256];
  __syncthreads();
  const int cw = P.W / SUB, ch = P.H / SUB;
  const int x = blockIdx.x * 64 + (threadIdx.x & 63), y = blockIdx.y * 4 + (threadIdx.x >> 6);
  if (x >= cw || y >= ch) return;
  const int v = reinterpret_cast<const uint16_t*>(P.src[C])[(size_t)y * P.srcStride[C] + x];
  int o = v;
  if (P.present[C]) {
    const int bx = x / BW, i = x - bx * BW;
    int g = fg_grain<C>(P, lut, x, y);
    if ((i == 0 && bx > 0) || (i == BW - 1 && bx + 1 < P.nbx)) g = (fg_grain<C>(P, lut, x - 1, y) + 3 * g + fg_grain<C>(P, lut, x + 1, y) + 2) >> 2;
    const int scale = lut[256 + ((v >> P.bs) & 0xff)];
    o = min(max(v + ((scale * g + (1 << (P.scaleShift - 1))) >> P.scaleShift), 0), 255 << P.bs);
  }
  P.dst[C][(size_t)y * P.dstStride[C] + x] = (int16_t)o;
}

// tables: device copies (pattern 64 KB, sLUT / pLUT 768 B each, lineSeeds); seeds: scratch of nbx * nby words
int launch_film_grain(const DevPlanes& src, const DevPlanes& dst, const b200_geom& g, const int8_t* pattern, const uint8_t* sLUT, const uint8_t* pLUT,
                      const uint32_t* lineSeeds, uint32_t* seeds, int scaleShift, const uint8_t present[3], cudaStream_t s, KHook* hook)
{
  FgParams P;
  for (int c = 0; c < 3; c++) { P.src[c] = src.p[c]; P.dst[c] = dst.p[c]; P.srcStride[c] = src.stride[c]; P.dstStride[c] = dst.stride[c]; P.present[c] = present[c]; }
  P.W = g.width; P.H = g.height; P.bs = g.bitDepth - 8; P.scaleShift = scaleShift; P.nbx = (g.width + 15) / 16;
  P.pattern = pattern; P.sLUT = sLUT; P.pLUT = pLUT; P.seeds = seeds;
  const int nby = (g.height + 15) / 16;
  fg_seed_kernel<<<(nby + 63) / 64, 64, 0, s>>>(lineSeeds, P.nbx, nby, seeds); hook_count(hook);
  fg_kernel<0><<<dim3((g.width + 63) / 64, (g.height + 3) / 4), 256, 0, s>>>(P); hook_count(hook);
  if (g.chromaFormat) {
    const dim3 grd((g.width / 2 + 63) / 64, (g.height / 2 + 3) / 4);
    fg_kernel<1><<<grd, 256, 0, s>>>(P); hook_count(hook);
    fg_kernel<2><<<grd, 256, 0, s>>>(P); hook_count(hook);
  }
  B200_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b200
