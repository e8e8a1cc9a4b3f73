// lmcs.cu — LMCS (luma mapping with chroma scaling) steps that are not fused into K1 / K2.
//
// Replaces (reference, source/Lib/CommonLib/Reshape.cpp): calculateChromaAdjVpduNei :192 + getPWLIdxInv :283 (one warp per VPDU),
// rspCtuBcw :377 -> applyLutCore Buffer.cpp:200 (whole luma plane, LUT in shared memory).  The forward map of the inter prediction
// (rspBufFwd :410 -> rspFwdCore Buffer.cpp:321) lives in K2's luma stores (lmcs_fwd below), the residual scaling (scaleSignal
// Buffer.cpp:412) in K1's chroma pass (lmcs_scale below).
#include "common.cuh"

namespace b200 {

// one warp per VPDU: lanes walk the 64 (or CTU-size) samples left of / above the CU that covers the VPDU's top-left sample
__global__ void __launch_bounds__(256) lmcs_vpdu_kernel(const int16_t* __restrict__ luma, int stride, int W, int H, int bitDepth, int numNeighbor,
                                                        const b200_lmcs* __restrict__ L, const b200_lmcs_vpdu* __restrict__ vpdus, int numVpdus, int* __restrict__ scale)
{
  const int v = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (v >= numVpdus) return;
  const int xPos = vpdus[v].x, yPos = vpdus[v].y, aL = vpdus[v].availLeft, aA = vpdus[v].availAbove;
  const int16_t* rec = luma + (size_t)yPos * stride + xPos;
  int sum = 0;
  for (int i = lane; i < numNeighbor; i += 32) {
    if (aL) { const int k = (yPos + i) >= H ? (H - yPos - 1) : i; sum += rec[-1 + (ptrdiff_t)k * stride]; }
    if (aA) { const int k = (xPos + i) >= W ? (W - xPos - 1) : i; sum += rec[-(ptrdiff_t)stride + k]; }
  }
#pragma unroll
  for (int m = 16; m; m >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, m);
  if (lane == 0) {
    const int l2 = 31 - __clz(numNeighbor), pelnum = (aL ? numNeighbor : 0) + (aA ? numNeighbor : 0);
    int lumaValue;
    if (pelnum == numNeighbor) lumaValue = (sum + (1 << (l2 - 1))) >> l2;
    else if (pelnum == 2 * numNeighbor) lumaValue = (sum + (1 << l2)) >> (l2 + 1);
    else lumaValue = 1 << (bitDepth - 1);
    int idx;
    for (idx = L->minBinIdx; idx <= L->maxBinIdx; idx++) if (lumaValue < L->reshapePivot[idx + 1]) break;
    scale[v] = L->chromaAdjHelpLUT[min(idx, 15)];
  }
}

// inverse map of the whole luma plane in place, 8 samples per thread
__global__ void __launch_bounds__(256) lmcs_inv_kernel(int16_t* __restrict__ luma, int stride, int W, int H, int bitDepth, const int16_t* __restrict__ lut)
{
  extern __shared__ int16_t sLut[];
  for (int i = threadIdx.x; i < (1 << bitDepth); i += 256) sLut[i] = lut[i];
  __syncthreads();
  const int x = (blockIdx.x * 32 + (threadIdx.x & 31)) * 8, y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= H) return;
  int16_t* p = luma + (size_t)y * stride + x;
  if (x + 8 <= W && !(stride & 7)) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    unsigned* w = reinterpret_cast<unsigned*>(&u);
#pragma unroll
    for (int k = 0; k < 4; k++) w[k] = (unsigned)(uint16_t)sLut[w[k] & 0xffff] | ((unsigned)(uint16_t)sLut[w[k] >> 16] << 16);
    *reinterpret_cast<uint4*>(p) = u;
  } else {
    for (int k = 0; k < 8 && x + k < W; k++) p[k] = sLut[(uint16_t)p[k]];
  }
}

// every VPDU record against lmcs_vpdu_problem (rules.cuh): error bit 16 of the PU meta block, read by b200_pic_run before lmcs_vpdu_kernel runs
__global__ void __launch_bounds__(256) lmcs_validate_kernel(const b200_lmcs_vpdu* __restrict__ vpdus, int numVpdus, const b200_geom g, int* meta)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < numVpdus && lmcs_vpdu_problem(vpdus[i], i, g)) atomicOr(&meta[LM_ERR], 16);
}

int launch_lmcs_validate(const b200_lmcs_vpdu* vpdus, const b200_geom& g, int* meta, cudaStream_t s, KHook* hook)
{
  const int vs = g.ctuSize == 128 ? 64 : g.ctuSize;
  const int n = ((g.width + vs - 1) / vs) * ((g.height + vs - 1) / vs);
  lmcs_validate_kernel<<<(n + 255) / 256, 256, 0, s>>>(vpdus, n, g, meta); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  return 0;
}

int launch_lmcs_vpdu(const LmcsLaunch& L, cudaStream_t s, KHook* hook)
{
  const int vs = L.geom.ctuSize == 128 ? 64 : L.geom.ctuSize;
  const int n = ((L.geom.width + vs - 1) / vs) * ((L.geom.height + vs - 1) / vs);
  hook_begin(hook, B200_KF_LMCS, s);
  lmcs_vpdu_kernel<<<(n + 7) / 8, 256, 0, s>>>(L.planes.p[0], L.planes.stride[0], L.geom.width, L.geom.height, L.geom.bitDepth, vs, L.lmcs, L.vpdus, n, L.scale); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  hook_end(hook, B200_KF_LMCS, s);
  return 0;
}

int launch_lmcs_inv(const LmcsLaunch& L, cudaStream_t s, KHook* hook)
{
  dim3 grd((L.geom.width + 255) / 256, (L.geom.height + 7) / 8);
  hook_begin(hook, B200_KF_LMCS, s);
  lmcs_inv_kernel<<<grd, 256, sizeof(int16_t) << L.geom.bitDepth, s>>>(L.planes.p[0], L.planes.stride[0], L.geom.width, L.geom.height, L.geom.bitDepth, L.invLut); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  hook_end(hook, B200_KF_LMCS, s);
  return 0;
}

}  // namespace b200
