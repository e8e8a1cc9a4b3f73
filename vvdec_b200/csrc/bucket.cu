// bucket.cu — device-side work-list bucketing.  The picture path copies the caller's PU / TU arrays as they are and does no per-record host work;
// two small kernels per array sort record indices into the lists the compute kernels walk:
//   MC tiles  (<=16x16 pieces of PUs): list = mode*4 + size class (mode 0 uni, 1 bi, 2 bi+BDOF, 3 DMVR; 32/64/128/256 samples), 16 = affine
//   TUs: list = size class (max dimension <= 8, 16, 32, 64)
// Order inside a list is arbitrary (atomics): tiles and TUs never overlap, so every order gives the same picture.
// Pass 1 counts (shared-memory histogram per CTA, one global atomic per list and CTA; the last CTA turns counts into offsets),
// pass 2 reserves a range per CTA and list and writes the entries.  Records that break a rule of rules.cuh raise bits in meta[LM_ERR] instead of faulting.
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
__device__ __forceinline__ PuHead pu_head(const b200_pu* pus, int i, const PuLimits lim)
{
  const b200_pu& p = pus[i];
  PuHead r; r.w = p.w; r.h = p.h; r.flags = p.flags; r.bi = p.refSlot[0] >= 0 && p.refSlot[1] >= 0; r.ok = !pu_problem(p, lim);
  return r;
}

__global__ void __launch_bounds__(256) mc_count_kernel(const b200_pu* __restrict__ pus, int numPus, int* meta, const PuLimits lim, int cap)
{
  __shared__ int h[MC_LISTS]; __shared__ int sLast;
  if (threadIdx.x < MC_LISTS) h[threadIdx.x] = 0;
  __syncthreads();
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < numPus) {
    const PuHead p = pu_head(pus, i, lim);
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

__global__ void __launch_bounds__(256) mc_scatter_kernel(const b200_pu* __restrict__ pus, int numPus, int* meta, uint32_t* __restrict__ tiles, const PuLimits lim)
{
  __shared__ int h[MC_LISTS], base[MC_LISTS];
  if (threadIdx.x < MC_LISTS) h[threadIdx.x] = 0;
  __syncthreads();
  const int i = blockIdx.x * 256 + threadIdx.x;
  PuHead p; p.ok = false;
  if (i < numPus) p = pu_head(pus, i, lim);
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

__device__ __forceinline__ int tu_class(const b200_tu* tus, int i, bool& ok, const TuLimits lim)
{
  const b200_tu& t = tus[i];
  ok = !tu_problem(t, lim);
  const int m = max(t.log2w, t.log2h);
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

int launch_mc_bucket(const b200_pu* pus, size_t numPus, uint32_t* tiles, size_t capTiles, int* meta, const b200_geom& g, int numSlots, int numWp, size_t numDmvr, cudaStream_t s, KHook* hook)
{
  const PuLimits lim = pu_limits(g, numSlots, numWp, numDmvr);
  B200_CUDA(cudaMemsetAsync(meta, 0, LM_INTS * sizeof(int), s));
  if (!numPus) return 0;
  const int grid = (int)((numPus + 255) / 256);
  mc_count_kernel<<<grid, 256, 0, s>>>(pus, (int)numPus, meta, lim, (int)capTiles); hook_count(hook);
  mc_scatter_kernel<<<grid, 256, 0, s>>>(pus, (int)numPus, meta, tiles, lim); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  return 0;
}

int launch_tu_bucket(const b200_tu* tus, size_t numTus, uint32_t* idx, int* meta, const b200_geom& g, size_t numCoefs, size_t numScaling, cudaStream_t s, KHook* hook)
{
  const TuLimits lim = tu_limits(g, numCoefs, numScaling);
  B200_CUDA(cudaMemsetAsync(meta, 0, LM_INTS * sizeof(int), s));
  if (!numTus) return 0;
  const int grid = (int)((numTus + 255) / 256);
  tu_count_kernel<<<grid, 256, 0, s>>>(tus, (int)numTus, meta, lim); hook_count(hook);
  tu_scatter_kernel<<<grid, 256, 0, s>>>(tus, (int)numTus, meta, idx, lim); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  return 0;
}

size_t mc_tile_capacity(const b200_geom& g, size_t numPus)
{
  // non-overlapping PUs of at least 4x4 samples; callers that pass overlapping PUs (unit tests) get numPus * 64 on top
  return (size_t)((g.width + 3) >> 2) * ((g.height + 3) >> 2) + numPus * 64;
}

// Per-CTU side information (SAO / ALF / slice index): every index the filter kernels use to address a table is range-checked here
// (error bit 4 of the PU meta block), so that a malformed record cannot make them read outside the uploaded arrays.
__global__ void __launch_bounds__(256) ctu_validate_kernel(const b200_sao_ctu* __restrict__ sao, const b200_alf_ctu* __restrict__ alf, const uint8_t* __restrict__ ctuSlice,
                                                           int nCtu, const CtuLimits lim, int* meta)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= nCtu) return;
  // SAO: every component's fields, those of 4:0:0 pictures included
  if ((sao && sao_ctu_problem(sao[i], 3)) || (alf && alf_ctu_problem(alf[i], i, lim)) || (ctuSlice && ctuSlice[i] >= lim.numLfSlices)) atomicOr(&meta[LM_ERR], 4);
}

int launch_ctu_validate(const b200_sao_ctu* sao, const b200_alf_ctu* alf, const uint8_t* ctuSlice, int nCtu, const CtuLimits& lim, int* meta, cudaStream_t s, KHook* hook)
{
  if (!nCtu || (!sao && !alf && !ctuSlice)) return 0;
  ctu_validate_kernel<<<(nCtu + 255) / 256, 256, 0, s>>>(sao, alf, ctuSlice, nCtu, lim, meta); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b200
