// lf_derive.cu — B200_PIC_DERIVE_LF: the deblocking edge grids derived on the device from CU / TU records (lf_derive.cuh holds the derivation, shared with the
// host).  On the context stream before K3: CU maps, motion field (over each CU's PU records), edge grids (luma-type CUs, then chroma-tree
// CUs), each a warp per CU record; the record check runs at upload.
#define VVC_TABLE_QUAL static __device__ const __align__(16)
#include "vvc_tables.h"
#include "common.cuh"
#include "lf_derive.cuh"

namespace b200 {

__global__ void lf_validate_kernel(const b200_lf_cu* cus, const b200_lf_tu* tus, const uint32_t* ctuCus, int nCtu, size_t numCus, LfLimits lim, int* meta)
{
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= nCtu) return;
  const uint32_t c0 = ctuCus[a], c1 = ctuCus[a + 1];
  bool bad = c0 > c1 || c1 > numCus || (a == nCtu - 1 && c1 != numCus) || (a == 0 && c0 != 0);
  for (uint32_t i = c0; i < c1 && !bad; i++) bad = lf_cu_problem(cus[i], tus, a, lim) != nullptr;
  if (bad) atomicOr(&meta[LM_ERR], LM_ERR_LF_RECORD);
}

// one warp per CU record (4 per CTA), its lanes over the CU's units
__global__ void lf_map_kernel(const LfDerive G, uint32_t* map0, uint32_t* map1, uint32_t numCus)
{
  const uint32_t i = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (i >= numCus) return;
  uint32_t* const maps[2] = {map0, map1};
  lf_map_cu(G, maps, i, threadIdx.x & 31, 32);
}

__global__ void lf_motion_kernel(const LfDerive G, uint32_t numCus)
{
  const uint32_t i = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (i < numCus) lf_cu_motion(G, i, kGeoParams, threadIdx.x & 31, 32);
}

// one warp per CU of channel type ch (luma-type CUs first, then chroma-tree CUs, lf_cu_runs): the three parts of lf_derive.cuh with a warp barrier between them
__global__ void lf_grid_kernel(const LfDerive G, const uint32_t* ctuCus, int nCtu, uint32_t numCus, int ch, bool anyDisabled)
{
  const uint32_t i = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= numCus || G.cus[i].chType != ch || !lf_cu_runs(G, i, ctuCus, nCtu, anyDisabled)) return;
  const bool refine = lf_cu_tu_edges(G, i, lane, 32);
  if (!refine) return;
  __syncwarp();
  if (lane == 0) lf_cu_sub_block_edges<0>(G, i);
  if (lane == 1) lf_cu_sub_block_edges<1>(G, i);
  __syncwarp();
  lf_cu_bs_walk(G, i, lane, 32);
}

int launch_lf_validate(const b200_lf_cu* cus, size_t numCus, const b200_lf_tu* tus, size_t numTus, const uint32_t* ctuCus, const b200_geom& g, int numSlices, int* meta, cudaStream_t s, KHook* hook)
{
  const int nCtu = ((g.width + g.ctuSize - 1) / g.ctuSize) * ((g.height + g.ctuSize - 1) / g.ctuSize);
  lf_validate_kernel<<<(nCtu + 127) / 128, 128, 0, s>>>(cus, tus, ctuCus, nCtu, numCus, lf_limits(g, numSlices, numTus), meta);
  hook_count(hook);
  B200_CUDA(cudaGetLastError());
  return 0;
}

int launch_lf_derive(const LfDeriveLaunch& L, cudaStream_t s, KHook* hook)
{
  const b200_geom& g = L.geom;
  const int W4 = g.width >> 2, H4 = g.height >> 2, nCtu = ((g.width + g.ctuSize - 1) / g.ctuSize) * ((g.height + g.ctuSize - 1) / g.ctuSize);
  const size_t n4 = (size_t)W4 * H4;
  LfDerive G{};
  G.W4 = W4; G.H4 = H4; G.ctuSize = g.ctuSize; G.chroma = g.chromaFormat; G.qpBdOffset2 = 12 * (g.bitDepth - 8);
  G.cus = L.cus; G.tus = L.tus; G.pus = L.pus; G.numPus = L.numPus; G.cuMap[0] = L.map[0]; G.cuMap[1] = L.map[1]; G.mi = L.mi;
  G.slices = L.slices; G.sliceB = L.sliceB; G.grid[0] = L.lfV; G.grid[1] = L.lfH;
  hook_begin(hook, B200_KF_LF_DERIVE, s);
  // entries no CU writes stay zero (the glue clears the reference's arrays the same way, LF_INIT)
  B200_CUDA(cudaMemsetAsync(L.map[0], 0xff, 2 * n4 * sizeof(uint32_t), s));
  B200_CUDA(cudaMemsetAsync(L.lfV, 0, n4 * sizeof(b200_lf_param), s));
  B200_CUDA(cudaMemsetAsync(L.lfH, 0, n4 * sizeof(b200_lf_param), s));
  const uint32_t n = (uint32_t)L.numCus;
  if (n) {
    const uint32_t blocks = (n + 3) / 4;
    lf_map_kernel<<<blocks, 128, 0, s>>>(G, L.map[0], L.map[1], n); hook_count(hook); B200_CUDA(cudaGetLastError());
    lf_motion_kernel<<<blocks, 128, 0, s>>>(G, n); hook_count(hook); B200_CUDA(cudaGetLastError());
    for (int ch = 0; ch < 2; ch++) { lf_grid_kernel<<<blocks, 128, 0, s>>>(G, L.ctuCus, nCtu, n, ch, L.anyDisabled); hook_count(hook); B200_CUDA(cudaGetLastError()); }
  }
  hook_end(hook, B200_KF_LF_DERIVE, s);
  return 0;
}

}  // namespace b200
