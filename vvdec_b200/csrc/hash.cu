// hash.cu — decoded-picture hash (DPH SEI check) on the device (SURVEY 8f-3): CRC and checksum of the three planes, so that a
// verify-only run moves 6 or 12 bytes per picture over PCIe instead of the frame.
// Replaces (reference, source/Lib/CommonLib/PicYuvMD5.cpp): compCRC :100-136 / calcCRC :138, compChecksum :152-177 / calcChecksum :179.
// (The MD5 variant, calcMD5 :198, is one serial chain per plane and is not offered here.)
//
// CRC: the reference shifts the message bits (per sample: low byte, then high byte when bitDepth > 8, MSB first) into a 16-bit
// register initialised to 0xffff with polynomial 0x1021, then 16 zero bits.  With R(M) = M(x) mod P that is
//     crc = ((0xffff * x^n  +  M(x)) * x^16) mod P ,  n = number of message bits,
// and M(x) = sum_j chunk_j(x) * x^(bits behind chunk j): every thread reduces one chunk, a warp tree joins 32 neighbours with
// constant multipliers, and one lane per warp raises x^(warp's bits) to the number of warps behind it.  Leading zero bits do not change
// M(x), so the message is padded at the FRONT to a whole number of warps and all chunks have the same length.
#include "common.cuh"

namespace b200 {

constexpr int HASH_CHUNK = 32;                 // samples per thread
constexpr int HASH_WARP  = HASH_CHUNK * 32;    // samples per warp

__host__ __device__ inline uint32_t crc_mulmod(uint32_t a, uint32_t b)      // a(x) * b(x) mod (x^16 + 0x1021), 16-bit operands
{
  uint32_t r = 0;
  for (int i = 15; i >= 0; i--) {
    r = ((r << 1) ^ ((r & 0x8000u) ? 0x11021u : 0u)) & 0xffffu;
    if ((b >> i) & 1u) r ^= a;
  }
  return r;
}
__host__ __device__ inline uint32_t crc_xpow(unsigned long long e)          // x^e mod P
{
  uint32_t r = 1, b = 2;
  while (e) { if (e & 1) r = crc_mulmod(r, b); b = crc_mulmod(b, b); e >>= 1; }
  return r;
}

struct HashParams { const int16_t* src; int stride, W, H, two; long long N, pad; uint32_t c[5]; uint32_t warpMul; uint32_t* out; };

__global__ void __launch_bounds__(256) crc_kernel(const HashParams P)
{
  __shared__ uint16_t T[256];                  // T[v] = v(x) * x^16 mod P: one byte per step
  { uint32_t r = threadIdx.x << 8; for (int k = 0; k < 8; k++) r = ((r << 1) ^ ((r & 0x8000u) ? 0x11021u : 0u)) & 0xffffu; T[threadIdx.x] = (uint16_t)r; }
  __syncthreads();
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long warpId = t >> 5, nWarps = (P.N + P.pad) / HASH_WARP;
  if (warpId >= nWarps) return;                // whole warps leave together
  long long i0 = t * HASH_CHUNK - P.pad;       // dense sample index of this chunk (negative: front padding)
  int n = HASH_CHUNK;
  if (i0 < 0) { n += (int)max(i0, (long long)-HASH_CHUNK); i0 = 0; }
  uint32_t r = 0;
  if (n > 0) {
    int y = (int)(i0 / P.W), x = (int)(i0 - (long long)y * P.W);
    const uint16_t* row = reinterpret_cast<const uint16_t*>(P.src) + (size_t)y * P.stride;
    for (int k = 0; k < n; k++) {
      const uint32_t v = row[x];
      r = (((r << 8) & 0xffffu) | (v & 0xffu)) ^ T[r >> 8];
      if (P.two) r = (((r << 8) & 0xffffu) | (v >> 8)) ^ T[r >> 8];
      if (++x == P.W) { x = 0; row += P.stride; }
    }
  }
#pragma unroll
  for (int k = 0; k < 5; k++) {                // join neighbours: left * x^(bits of the right run) + right
    const uint32_t right = __shfl_down_sync(0xffffffffu, r, 1 << k);
    r = crc_mulmod(r, P.c[k]) ^ right;
  }
  if ((threadIdx.x & 31) == 0) {
    uint32_t m = 1, b = P.warpMul; long long e = nWarps - 1 - warpId;
    while (e) { if (e & 1) m = crc_mulmod(m, b); b = crc_mulmod(b, b); e >>= 1; }
    atomicXor(P.out, crc_mulmod(r, m));
  }
}

__global__ void __launch_bounds__(256) checksum_kernel(const HashParams P)
{
  const int x0 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 4, y = blockIdx.y * 8 + (threadIdx.x >> 5);
  uint32_t s = 0;
  if (x0 < P.W && y < P.H) {
    const uint16_t* p = reinterpret_cast<const uint16_t*>(P.src) + (size_t)y * P.stride + x0;
#pragma unroll
    for (int k = 0; k < 4; k++) if (x0 + k < P.W) {
      const uint32_t x = x0 + k, mask = ((x & 0xff) ^ (y & 0xff) ^ (x >> 8) ^ (y >> 8)) & 0xff, v = p[k];
      s += (v & 0xff) ^ mask;
      if (P.two) s += (v >> 8) ^ mask;
    }
  }
  for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  __shared__ uint32_t part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) { uint32_t a = 0; for (int k = 0; k < 8; k++) a += part[k]; if (a) atomicAdd(P.out, a); }
}

// digest bytes in the order PictureHash::hash holds them: per component CRC hi, lo  |  checksum big endian
__global__ void hash_finish_kernel(const uint32_t* acc, int method, int nPl, uint32_t initMul0, uint32_t initMul1, uint8_t* out)
{
  const int c = threadIdx.x;
  if (c >= nPl) return;
  if (method == B200_HASH_CRC) {
    uint32_t r = acc[c] ^ crc_mulmod(0xffffu, c ? initMul1 : initMul0);
    r = crc_mulmod(r, 0x1021u);                // * x^16 mod P (x^16 = 0x1021 mod P)
    out[2 * c] = (uint8_t)(r >> 8); out[2 * c + 1] = (uint8_t)r;
  } else {
    const uint32_t v = acc[c];
    out[4 * c] = (uint8_t)(v >> 24); out[4 * c + 1] = (uint8_t)(v >> 16); out[4 * c + 2] = (uint8_t)(v >> 8); out[4 * c + 3] = (uint8_t)v;
  }
}

// acc: 3 zero-initialised words (device), digest: 12 bytes (device)
int launch_hash(const DevPlanes& src, const b200_geom& g, int method, uint32_t* acc, uint8_t* digest, cudaStream_t s, KHook* hook)
{
  const int nPl = g.chromaFormat ? 3 : 1, two = g.bitDepth > 8;
  uint32_t initMul[2] = {1, 1};
  for (int c = 0; c < nPl; c++) {
    HashParams P; P.src = src.p[c]; P.stride = src.stride[c]; P.W = c ? g.width >> 1 : g.width; P.H = c ? g.height >> 1 : g.height; P.two = two;
    P.N = (long long)P.W * P.H; P.pad = (HASH_WARP - P.N % HASH_WARP) % HASH_WARP; P.out = acc + c;
    if (method == B200_HASH_CRC) {
      const unsigned long long bitsPerSample = two ? 16 : 8;
      for (int k = 0; k < 5; k++) P.c[k] = crc_xpow(bitsPerSample * HASH_CHUNK << k);
      P.warpMul = crc_xpow(bitsPerSample * HASH_WARP);
      if (c < 2) initMul[c] = crc_xpow(bitsPerSample * (unsigned long long)P.N);
      const long long threads = (P.N + P.pad) / HASH_CHUNK;
      crc_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(P); hook_count(hook);
    } else {
      for (int k = 0; k < 5; k++) P.c[k] = 0; P.warpMul = 0;
      dim3 grd((P.W + 127) / 128, (P.H + 7) / 8);
      checksum_kernel<<<grd, 256, 0, s>>>(P); hook_count(hook);
    }
  }
  hash_finish_kernel<<<1, 32, 0, s>>>(acc, method, nPl, initMul[0], initMul[1], digest); hook_count(hook);
  B200_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b200
