// bucket.cu — device-side work-list bucketing.  The host copies the caller's PU / TU arrays as they are and does no per-record work;
// two small kernels per array sort record indices into the lists the compute kernels walk:
//   MC tiles  (<=16x16 pieces of PUs): list = mode*4 + size class (mode 0 uni, 1 bi, 2 bi+BDOF, 3 DMVR; 32/64/128/256 samples), 16 = affine
//   TUs: list = size class (max dimension <= 8, 16, 32, 64)
// Order inside a list is arbitrary (atomics): tiles and TUs never overlap, so every order gives the same picture.
// Pass 1 counts (shared-memory histogram per CTA, one global atomic per list and CTA; the last CTA turns counts into offsets),
// pass 2 reserves a range per CTA and list and writes the entries.  Invalid records raise bits in meta[LM_ERR] instead of faulting.
#include "common.cuh"

namespace b200 {

__device__ __forceinline__ int mc_list_of(int w, int h, int flags, bool bi, int tx, int ty)
{
  if (flags & B200_PU_AFFINE) return 16;
  const int mode = (flags & B200_PU_GEO) ? 1 : (flags & B200_PU_DMVR) ? 3 : (bi && (flags & B200_PU_BDOF)) ? 2 : bi ? 1 : 0;
  const int tw = min(16, w - tx * 16), th = min(16, h - ty * 16), n = tw * th;
  return mode * 4 + (n <= 32 ? 0 : n <= 64 ? 1 : n <= 128 ? 2 : 3);
}

struct PuHead { int w, h, flags; bool bi, ok; };
struct PuLimits { int slotsBd, W, H; unsigned numDmvr; };   // slotsBd = numSlots | bitDepth << 8 | numWp << 16
__device__ __forceinline__ PuHead pu_head(const b200_pu* pus, int i, const PuLimits lim)
{
  const int slotsBd = lim.slotsBd;
  const b200_pu& p = pus[i];
  PuHead r; r.w = p.w; r.h = p.h; r.flags = p.flags;
  const int s0 = p.refSlot[0], s1 = p.refSlot[1], numSlots = slotsBd & 0xff, bitDepth = (slotsBd >> 8) & 0xff, numWp = slotsBd >> 16;
  r.bi = s0 >= 0 && s1 >= 0;
  // sides are multiples of 4 (CUs: powers of two; SbTMVP runs: multiples of 8) whose 16-sample tiles end in a 4, 8 or 16 piece: mc_tile maps threads to
  // samples with tw - 1 masks and log2(tw) shifts, so a 12-sample piece (sides 12, 28, 44, ...) would filter wrong columns and store below the tile
  r.ok = s0 < numSlots && s1 < numSlots && (s0 >= 0 || s1 >= 0) && r.w >= 4 && r.h >= 4 && r.w <= 128 && r.h <= 128 && !(r.w & 3) && !(r.h & 3) &&
         (r.w & 15) != 12 && (r.h & 15) != 12;
  // the block must lie inside the picture on the 4x4 grid (kernels write every sample of it), DMVR deltas inside the output array
  if ((p.x & 3) || (p.y & 3) || p.x + r.w > lim.W || p.y + r.h > lim.H) r.ok = false;
  if ((r.flags & B200_PU_DMVR) && (unsigned long long)p.dmvrOff + (unsigned)(max(1, r.w >> 4) * max(1, r.h >> 4)) > lim.numDmvr) r.ok = false;
  // BDOF / DMVR blocks are at least 8x8 with 128 samples (conditions at InterPrediction.cpp:1372-1420); DMVR also needs both lists and
  // is never affine.  A BDOF flag on a uni-predicted or affine PU is ignored, as the launch-side classification always did.
  const bool big = r.w >= 8 && r.h >= 8 && r.w * r.h >= 128, aff = r.flags & B200_PU_AFFINE;
  if ((r.flags & B200_PU_DMVR) && (!r.bi || !big || aff)) r.ok = false;
  if ((r.flags & B200_PU_BDOF) && r.bi && !aff && !big) r.ok = false;
  if ((r.flags & B200_PU_DMVR) && bitDepth > 10) r.ok = false;
  // GEO (InterPrediction.cpp:1461): two partitions = both 'lists' set, 8..64 luma samples per side, never with another tool; bcwW1 = split direction
  if (r.flags & B200_PU_GEO) {
    if (!r.bi || r.w < 8 || r.h < 8 || r.w > 64 || r.h > 64 || (r.w & (r.w - 1)) || (r.h & (r.h - 1)) || (r.flags & (B200_PU_DMVR | B200_PU_BDOF | B200_PU_AFFINE)) || p.wpIdx || (uint8_t)p.bcwW1 > 63) r.ok = false;
  }
  // explicit weights: the entry must exist; the reference never combines them with BDOF / DMVR / BCW (InterPrediction.cpp:733, :1406-1420)
  const int wpIdx = p.wpIdx;
  if (wpIdx && (wpIdx > numWp || (r.flags & B200_PU_DMVR) || ((r.flags & B200_PU_BDOF) && r.bi && !aff) || p.bcwW1 != 4) && !(r.flags & B200_PU_GEO)) r.ok = false;   // DMVR is defined for bit depths <= 10 only (as in the reference)
  return r;
}

__global__ void __launch_bounds__(256) mc_count_kernel(const b200_pu* __restrict__ pus, int numPus, int* meta, const PuLimits numSlots, int cap)
{
  __shared__ int h[MC_LISTS]; __shared__ int sLast;
  if (threadIdx.x < MC_LISTS) h[threadIdx.x] = 0;
  __syncthreads();
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < numPus) {
    const PuHead p = pu_head(pus, i, numSlots);
    if (!p.ok) atomicOr(&meta[LM_ERR], 1);
    else for (int ty = 0; ty * 16 < p.h; ty++) for (int tx = 0; tx * 16 < p.w; tx++) atomicAdd(&h[mc_list_of(p.w, p.h, p.flags, p.bi, tx, ty)], 1);
  }
  __syncthreads();
  if (threadIdx.x < MC_LISTS && h[threadIdx.x]) atomicAdd(&meta[LM_CNT + threadIdx.x], h[threadIdx.x]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) sLast = atomicAdd(&meta[LM_DONE], 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (sLast && threadIdx.x == 0) {
    __threadfence();
    int o = 0;
    for (int l = 0; l < MC_LISTS; l++) { const int c = atomicAdd(&meta[LM_CNT + l], 0); meta[LM_OFF + l] = o; meta[LM_CUR + l] = 0; o += c; }
    if (o > cap) { atomicOr(&meta[LM_ERR], 2); for (int l = 0; l < MC_LISTS; l++) meta[LM_CNT + l] = 0; }
  }
}

__global__ void __launch_bounds__(256) mc_scatter_kernel(const b200_pu* __restrict__ pus, int numPus, int* meta, uint32_t* __restrict__ tiles, const PuLimits numSlots)
{
  __shared__ int h[MC_LISTS], base[MC_LISTS];
  if (threadIdx.x < MC_LISTS) h[threadIdx.x] = 0;
  __syncthreads();
  const int i = blockIdx.x * 256 + threadIdx.x;
  PuHead p; p.ok = false;
  if (i < numPus) p = pu_head(pus, i, numSlots);
  if (meta[LM_ERR] & 2) return;                               // overflow: nothing is written, nothing will be run
  if (p.ok) for (int ty = 0; ty * 16 < p.h; ty++) for (int tx = 0; tx * 16 < p.w; tx++) atomicAdd(&h[mc_list_of(p.w, p.h, p.flags, p.bi, tx, ty)], 1);
  __syncthreads();
  if (threadIdx.x < MC_LISTS) { const int c = h[threadIdx.x]; base[threadIdx.x] = meta[LM_OFF + threadIdx.x] + (c ? atomicAdd(&meta[LM_CUR + threadIdx.x], c) : 0); h[threadIdx.x] = 0; }
  __syncthreads();
  if (p.ok) for (int ty = 0; ty * 16 < p.h; ty++) for (int tx = 0; tx * 16 < p.w; tx++) {
    const int l = mc_list_of(p.w, p.h, p.flags, p.bi, tx, ty);
    tiles[base[l] + atomicAdd(&h[l], 1)] = ((uint32_t)i << 6) | (ty << 3) | tx;
  }
}

struct TuLimits { int W, H, chroma; unsigned numCoefs, numScaling; };
__device__ __forceinline__ int tu_class(const b200_tu* tus, int i, bool& ok, const TuLimits lim)
{
  const b200_tu& t = tus[i];
  const int l2w = t.log2w, l2h = t.log2h, m = max(l2w, l2h);
  ok = m <= 6 && t.comp < 3;
  // one-sample-wide / -high blocks exist only as luma sub-partitions of an ISP CU (4xN, N >= 16 and the transpose): regular transform, no LFNST
  if ((l2w == 0 || l2h == 0) && (t.comp != 0 || m < 4 || l2w == l2h || t.lfnst || t.ict || (t.flags & (B200_TU_TS | B200_TU_BDPCM_H | B200_TU_BDPCM_V)))) ok = false;
  if (ok) {
    // inside its plane (the joint-CbCr partner plane has the same geometry), level corner and scaling table inside their arrays
    const int w = 1 << l2w, h = 1 << l2h, pw = t.comp ? lim.W >> 1 : lim.W, ph = t.comp ? lim.H >> 1 : lim.H;
    const bool ts = t.flags & B200_TU_TS;
    if ((t.comp && !lim.chroma) || t.x + w > pw || t.y + h > ph || t.maxX >= w || t.maxY >= h || (!ts && (t.maxX >= 32 || t.maxY >= 32))) ok = false;
    if ((unsigned long long)t.coefOff + (unsigned)((t.maxX + 1) * (t.maxY + 1)) > lim.numCoefs) ok = false;
    if ((t.flags & B200_TU_SCALING) && (unsigned long long)t.slOff + (unsigned)(w * h) > lim.numScaling) ok = false;
    if (t.inBits < 1 || t.inBits > 32 || t.rightShift < -31 || t.rightShift > 31) ok = false;
    // transform skip / BDPCM blocks are at most 32 wide (sps log2MaxTransformSkipBlockSize <= 5): K1 keeps them in the 32x32 working set of their class;
    // BDPCM accumulates over the whole block, so its level corner is the block
    const bool bdpcm = t.flags & (B200_TU_BDPCM_H | B200_TU_BDPCM_V);
    if ((ts || bdpcm) && (w > 32 || h > 32)) ok = false;
    if (bdpcm && (!ts || t.maxX != w - 1 || t.maxY != h - 1 || (t.flags & (B200_TU_BDPCM_H | B200_TU_BDPCM_V)) == (B200_TU_BDPCM_H | B200_TU_BDPCM_V))) ok = false;
    // LFNST: index 1 or 2, no stray bits, at least 4x4, never with transform skip (the kernel indexes kLfnst* with it)
    if (t.lfnst && ((t.lfnst & 3) < 1 || (t.lfnst & 3) > 2 || (t.lfnst & 0xe0) || ts || w < 4 || h < 4)) ok = false;
    // joint CbCr writes the partner chroma plane at the same position
    if (t.ict && (t.comp == 0 || !lim.chroma || t.ict < -3 || t.ict > 3)) ok = false;
  }
  return m <= 3 ? 0 : m == 4 ? 1 : m == 5 ? 2 : 3;
}

__global__ void __launch_bounds__(256) tu_count_kernel(const b200_tu* __restrict__ tus, int numTus, int* meta, const TuLimits lim)
{
  __shared__ int h[K1_LISTS]; __shared__ int sLast;
  if (threadIdx.x < K1_LISTS) h[threadIdx.x] = 0;
  __syncthreads();
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < numTus) { bool ok; const int c = tu_class(tus, i, ok, lim); if (ok) atomicAdd(&h[c], 1); else atomicOr(&meta[LM_ERR], 1); }
  __syncthreads();
  if (threadIdx.x < K1_LISTS && h[threadIdx.x]) atomicAdd(&meta[LM_CNT + threadIdx.x], h[threadIdx.x]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) sLast = atomicAdd(&meta[LM_DONE], 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (sLast && threadIdx.x == 0) {
    __threadfence();
    int o = 0;
    for (int l = 0; l < K1_LISTS; l++) { const int c = atomicAdd(&meta[LM_CNT + l], 0); meta[LM_OFF + l] = o; meta[LM_CUR + l] = 0; o += c; }
  }
}

__global__ void __launch_bounds__(256) tu_scatter_kernel(const b200_tu* __restrict__ tus, int numTus, int* meta, uint32_t* __restrict__ idx, const TuLimits lim)
{
  __shared__ int h[K1_LISTS], base[K1_LISTS];
  if (threadIdx.x < K1_LISTS) h[threadIdx.x] = 0;
  __syncthreads();
  const int i = blockIdx.x * 256 + threadIdx.x;
  bool ok = false; int c = 0, my = 0;
  if (i < numTus) c = tu_class(tus, i, ok, lim);
  if (ok) my = atomicAdd(&h[c], 1);
  __syncthreads();
  if (threadIdx.x < K1_LISTS) { const int n = h[threadIdx.x]; base[threadIdx.x] = meta[LM_OFF + threadIdx.x] + (n ? atomicAdd(&meta[LM_CUR + threadIdx.x], n) : 0); }
  __syncthreads();
  if (ok) idx[base[c] + my] = (uint32_t)i;
}

int launch_mc_bucket(const b200_pu* pus, size_t numPus, uint32_t* tiles, size_t capTiles, int* meta, const b200_geom& g, int numSlotsIn, int numWp, size_t numDmvr, cudaStream_t s)
{
  PuLimits numSlots; numSlots.slotsBd = numSlotsIn | (g.bitDepth << 8) | (numWp << 16); numSlots.W = g.width; numSlots.H = g.height;
  numSlots.numDmvr = (unsigned)(numDmvr > 0xffffffffu ? 0xffffffffu : numDmvr);
  B200_CUDA(cudaMemsetAsync(meta, 0, LM_INTS * sizeof(int), s));
  if (!numPus) return 0;
  const int grid = (int)((numPus + 255) / 256);
  mc_count_kernel<<<grid, 256, 0, s>>>(pus, (int)numPus, meta, numSlots, (int)capTiles);
  mc_scatter_kernel<<<grid, 256, 0, s>>>(pus, (int)numPus, meta, tiles, numSlots);
  B200_CUDA(cudaGetLastError());
  return 0;
}

int launch_tu_bucket(const b200_tu* tus, size_t numTus, uint32_t* idx, int* meta, const b200_geom& g, size_t numCoefs, size_t numScaling, cudaStream_t s)
{
  TuLimits lim; lim.W = g.width; lim.H = g.height; lim.chroma = g.chromaFormat != 0;
  lim.numCoefs = (unsigned)(numCoefs > 0xffffffffu ? 0xffffffffu : numCoefs); lim.numScaling = (unsigned)(numScaling > 0xffffffffu ? 0xffffffffu : numScaling);
  B200_CUDA(cudaMemsetAsync(meta, 0, LM_INTS * sizeof(int), s));
  if (!numTus) return 0;
  const int grid = (int)((numTus + 255) / 256);
  tu_count_kernel<<<grid, 256, 0, s>>>(tus, (int)numTus, meta, lim);
  tu_scatter_kernel<<<grid, 256, 0, s>>>(tus, (int)numTus, meta, idx, lim);
  B200_CUDA(cudaGetLastError());
  return 0;
}

size_t mc_tile_capacity(const b200_geom& g, size_t numPus)
{
  // non-overlapping PUs of at least 4x4 samples; callers that pass overlapping PUs (unit tests) get numPus * 64 on top
  return (size_t)((g.width + 3) >> 2) * ((g.height + 3) >> 2) + numPus * 64;
}

// Per-CTU side information (SAO / ALF / slice index): every index the filter kernels use to address a table is range-checked here
// (error bit 4 of the PU meta block), so that a malformed record cannot make them read outside the uploaded arrays.  ALF records also follow the
// rule b200_alf_picture checks on the host: no undefined enable bit, PAD_TL / PAD_BR only with both adjacent sides readable and inside the CTU grid,
// PAD_WIDE only without CC-ALF on that component.
__global__ void __launch_bounds__(256) ctu_validate_kernel(const b200_sao_ctu* __restrict__ sao, const b200_alf_ctu* __restrict__ alf, const uint8_t* __restrict__ ctuSlice,
                                                           int nCtu, const CtuLimits lim, int* meta)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= nCtu) return;
  bool ok = true;
  if (sao) for (int c = 0; c < 3; c++) { const int t = sao[i].type[c]; if (t != B200_SAO_OFF && (t > B200_SAO_BO || (t == B200_SAO_BO && sao[i].band[c] > 31))) ok = false; }
  if (alf) {
    const b200_alf_ctu a = alf[i];
    if ((a.enable[0] & 1) && a.lumaSet >= lim.numLumaSets) ok = false;
    for (int c = 0; c < 2; c++) {
      if ((a.enable[1 + c] & 1) && a.chromaAlt[c] >= lim.numChromaAlts) ok = false;
      if (a.ccIdx[c] > lim.numCc[c]) ok = false;
      if ((a.enable[1 + c] & ~3) || ((a.enable[1 + c] & B200_ALF_PAD_WIDE) && a.ccIdx[c])) ok = false;
    }
    const int f = a.enable[0], cx = i % lim.ctusW, cy = i / lim.ctusW;
    if (f & ~0x7f) ok = false;
    if ((f & B200_ALF_PAD_TL) && ((f & (B200_ALF_CLIP_TOP | B200_ALF_CLIP_LEFT)) || !cx || !cy)) ok = false;
    if ((f & B200_ALF_PAD_BR) && ((f & (B200_ALF_CLIP_BOTTOM | B200_ALF_CLIP_RIGHT)) || cx == lim.ctusW - 1 || cy == lim.ctusH - 1)) ok = false;
  }
  if (ctuSlice && ctuSlice[i] >= lim.numLfSlices) ok = false;
  if (!ok) atomicOr(&meta[LM_ERR], 4);
}

int launch_ctu_validate(const b200_sao_ctu* sao, const b200_alf_ctu* alf, const uint8_t* ctuSlice, int nCtu, const CtuLimits& lim, int* meta, cudaStream_t s)
{
  if (!nCtu || (!sao && !alf && !ctuSlice)) return 0;
  ctu_validate_kernel<<<(nCtu + 255) / 256, 256, 0, s>>>(sao, alf, ctuSlice, nCtu, lim, meta);
  B200_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b200
