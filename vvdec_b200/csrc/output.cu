// output.cu — output-format conversion on the device (SURVEY 8f-3), so that the D2H copy moves 5/8 (pyuv) or 1/2 (8 bit) of the bytes.
// Replaces (reference, source/App/vvdecapp/vvdecHelper.h): _writeComponentToFile :63 — the 8-bit narrowing loop :86-104 and the
// packed-yuv loop :115-128 (4 samples -> 5 bytes, little endian: s0 | s1<<10 | s2<<20 | s3<<30).
#include "common.cuh"

namespace b200 {

// one thread per 8 samples (two 5-byte groups = five 16-bit stores; rows are W*5/4 bytes, W % 4 == 0 -> 2-byte aligned groups of 8)
__global__ void __launch_bounds__(256) pack_pyuv_kernel(const int16_t* __restrict__ src, int stride, int W, int H, uint8_t* __restrict__ dst)
{
  const int x = (blockIdx.x * 32 + (threadIdx.x & 31)) * 8, y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= H) return;
  const uint16_t* p = reinterpret_cast<const uint16_t*>(src) + (size_t)y * stride + x;
  uint8_t* o = dst + (size_t)y * (W / 4 * 5) + x / 4 * 5;
  const unsigned long long g0 = (unsigned long long)p[0] | ((unsigned long long)p[1] << 10) | ((unsigned long long)p[2] << 20) | ((unsigned long long)p[3] << 30);
  const bool two = x + 8 <= W;
  const unsigned long long g1 = two ? (unsigned long long)p[4] | ((unsigned long long)p[5] << 10) | ((unsigned long long)p[6] << 20) | ((unsigned long long)p[7] << 30) : 0;
  if (two && !(W & 7)) {                                       // rows of W*5/4 bytes are even and x/4*5 is a multiple of 10: 16-bit stores
    uint16_t* o2 = reinterpret_cast<uint16_t*>(o);
    o2[0] = (uint16_t)g0; o2[1] = (uint16_t)(g0 >> 16); o2[2] = (uint16_t)(((g0 >> 32) & 0xff) | ((g1 & 0xff) << 8));
    o2[3] = (uint16_t)(g1 >> 8); o2[4] = (uint16_t)(g1 >> 24);
  } else {                                                     // widths that are 4 mod 8 (chroma of W = 8 mod 16): byte stores
    o[0] = (uint8_t)g0; o[1] = (uint8_t)(g0 >> 8); o[2] = (uint8_t)(g0 >> 16); o[3] = (uint8_t)(g0 >> 24); o[4] = (uint8_t)(g0 >> 32);
    if (two) { o[5] = (uint8_t)g1; o[6] = (uint8_t)(g1 >> 8); o[7] = (uint8_t)(g1 >> 16); o[8] = (uint8_t)(g1 >> 24); o[9] = (uint8_t)(g1 >> 32); }
  }
}

__global__ void __launch_bounds__(256) narrow8_kernel(const int16_t* __restrict__ src, int stride, int W, int H, int shift, uint8_t* __restrict__ dst)
{
  const int x = (blockIdx.x * 32 + (threadIdx.x & 31)) * 4, y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= W || y >= H) return;
  const uint16_t* p = reinterpret_cast<const uint16_t*>(src) + (size_t)y * stride + x;
  uint8_t* o = dst + (size_t)y * W + x;
#pragma unroll
  for (int k = 0; k < 4; k++) if (x + k < W) o[k] = (uint8_t)(p[k] >> shift);
}

int launch_pack(const DevPlanes& src, const b200_geom& g, int fmt, uint8_t* const dst[3], cudaStream_t s, KHook* hook)
{
  for (int c = 0; c < (g.chromaFormat ? 3 : 1); c++) {
    const int W = c ? g.width >> 1 : g.width, H = c ? g.height >> 1 : g.height;
    if (fmt == B200_OUT_PYUV) { dim3 grd((W + 255) / 256, (H + 7) / 8); pack_pyuv_kernel<<<grd, 256, 0, s>>>(src.p[c], src.stride[c], W, H, dst[c]); hook_count(hook); }
    else                      { dim3 grd((W + 127) / 128, (H + 7) / 8); narrow8_kernel<<<grd, 256, 0, s>>>(src.p[c], src.stride[c], W, H, g.bitDepth - 8, dst[c]); hook_count(hook); }
  }
  B200_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b200
