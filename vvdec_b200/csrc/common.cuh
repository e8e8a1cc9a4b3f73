// common.cuh — shared device/host helpers for the sm_90a kernels of vvdec_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>
#include "../../include/vvdec_b200.h"
#include "rules.cuh"

namespace b200 {

void set_error(const char* fmt, ...);

// A failed call is reported through the return code, and its error is consumed: the runtime keeps one last error per thread for the whole process, so a
// failure a caller handles (b200_host_register on an already registered range: the glue then uses the memory unpinned) must not resurface in a later,
// unrelated cudaGetLastError() check.  Sticky errors stay visible to the next call regardless.
#define B200_CUDA(call)                                                                         \
  do {                                                                                          \
    cudaError_t e_ = (call);                                                                    \
    if (e_ != cudaSuccess) {                                                                    \
      b200::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));     \
      (void)cudaGetLastError();                                                                 \
      return B200_ERR_CUDA;                                                                     \
    }                                                                                           \
  } while (0)

#define B200_CHECK(cond, ...)                                    \
  do {                                                           \
    if (!(cond)) { b200::set_error(__VA_ARGS__); return B200_ERR_PARAM; } \
  } while (0)

__device__ __forceinline__ int clip3(int lo, int hi, int v) { return min(max(v, lo), hi); }
__device__ __forceinline__ int clip16(int v) { return min(max(v, -32768), 32767); }

// Four int16 samples as one 8-byte word pair (K4 and K5 move 4 samples per thread)
__device__ __forceinline__ void unpack4(const uint2 u, int* d) { d[0] = (int)(int16_t)(u.x & 0xffff); d[1] = (int)(int16_t)(u.x >> 16); d[2] = (int)(int16_t)(u.y & 0xffff); d[3] = (int)(int16_t)(u.y >> 16); }
__device__ __forceinline__ uint2 pack4(const int* v)
{
  uint2 o;
  o.x = (unsigned)(v[0] & 0xffff) | ((unsigned)v[1] << 16);
  o.y = (unsigned)(v[2] & 0xffff) | ((unsigned)v[3] << 16);
  return o;
}

// Asynchronous global -> shared copies of 4, 8 and 16 bytes (LDGSTS): a CTA issues its whole footprint without waiting on any load, then waits once.
// 16-byte copies bypass L1 (.cg); the smaller sizes only exist cached (.ca).
__device__ __forceinline__ void cp_async4(void* smemDst, const void* gmemSrc)
{
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" :: "r"((unsigned)__cvta_generic_to_shared(smemDst)), "l"(gmemSrc));
}
__device__ __forceinline__ void cp_async8(void* smemDst, const void* gmemSrc)
{
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" :: "r"((unsigned)__cvta_generic_to_shared(smemDst)), "l"(gmemSrc));
}
__device__ __forceinline__ void cp_async16(void* smemDst, const void* gmemSrc)
{
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"((unsigned)__cvta_generic_to_shared(smemDst)), "l"(gmemSrc));
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// LMCS forward map of one predicted luma sample (rspFwdCore, reference CommonLib/Buffer.cpp:321); L points at the uploaded b200_lmcs
__device__ __forceinline__ int lmcs_fwd(const b200_lmcs* __restrict__ L, int log2OrgCW, int v, int pmax)
{
  const int idx = v >> log2OrgCW;
  return clip3(0, pmax, (int)__ldg(&L->reshapePivot[idx]) + (((int)__ldg(&L->fwdScaleCoef[idx]) * (v - (int)__ldg(&L->inputPivot[idx])) + (1 << 10)) >> 11));
}
// LMCS chroma residual scaling of one sample (AreaBuf<Pel>::scaleSignal, Buffer.cpp:412)
__device__ __forceinline__ int lmcs_scale(int r, int scale, int maxAbs)
{
  r = clip3(-maxAbs - 1, maxAbs, r);
  const int a = abs(r), v = (a * scale + (1 << 10)) >> 11;
  return clip16(r >= 0 ? v : -v);
}

// Grow-only device scratch buffer.
struct DevBuf {
  void*  p   = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + (bytes >> 2) + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) -> %s", want, cudaGetErrorString(e)); return B200_ERR_CUDA; }
    cap = want;
    return 0;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
  ~DevBuf() { if (p) cudaFree(p); }
};

// Device-resident picture planes (int16, no margins; kernels clamp coordinates).
struct DevPlanes {
  int16_t* p[3] = {nullptr, nullptr, nullptr};
  int      stride[3] = {0, 0, 0};
};

// A picture buffer holds Y | Cb | Cr, each plane at a 256-byte boundary (4:0:0: no chroma planes).
inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }
inline size_t plane_bytes(const b200_geom& g, int k) { return (size_t)g.stride[k] * (k ? g.height >> 1 : g.height) * 2; }
inline size_t plane_span(const b200_geom& g, int k) { return k == 0 || g.chromaFormat ? align256(plane_bytes(g, k)) : 0; }
inline size_t pic_bytes(const b200_geom& g) { return plane_span(g, 0) + plane_span(g, 1) + plane_span(g, 2); }
inline DevPlanes pic_planes(void* buf, const b200_geom& g)
{
  DevPlanes d; char* b = static_cast<char*>(buf);
  for (int k = 0; k < 3; k++) { d.p[k] = reinterpret_cast<int16_t*>(b); d.stride[k] = g.stride[k]; b += plane_span(g, k); }
  return d;
}

// A contiguous copy between caller memory and the device; a caller array that starts in a page registered for another array goes through a pinned
// staging copy (picture.cu: copy2d_host).
int copy2d_host(void* dst, size_t dpitch, const void* src, size_t spitch, size_t wBytes, size_t h, cudaMemcpyKind kind, cudaStream_t s);
inline int copy_host(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t s) { return copy2d_host(dst, bytes, src, bytes, bytes, 1, kind, s); }

// The device inputs of one call, laid out in one buffer.  add() starts an entry: an element count, a host source (copied) or none (device scratch), and
// the view that receives the entry's device address (null when the entry is empty).  pack() puts a further array into the last entry, right behind the
// previous one.  Every entry takes align256(bytes + 16).  commit() reserves the buffer, fills every view and enqueues the copies on the stream.  A part
// copies at most its span (stage_picture: the plane, into its 256-byte aligned span) and nothing when it has no space.
struct Staging {
  struct Part { void* view; void (*set)(void*, char*); const void* src; size_t copy, off, span; };
  std::vector<Part> parts;
  size_t top = 0, used = 0; bool open = false;   // end of the closed entries; bytes of the open one
  template <class V> static void set_view(void* v, char* p) { *static_cast<V**>(v) = reinterpret_cast<V*>(p); }
  template <class V> void put(V** view, const void* src, size_t copy, size_t span, bool entry)
  {
    if (entry) { if (open) top += align256(used + 16); used = 0; open = true; }
    parts.push_back({view, &set_view<V>, src, src && span ? std::min(copy, span) : 0, top + used, span}); used += span;
  }
  template <class V> void add(V** view, const void* src, size_t n) { put(view, src, n * sizeof(V), n * sizeof(V), true); }
  template <class V> void pack(V** view, const void* src, size_t n) { put(view, src, n * sizeof(V), n * sizeof(V), false); }
  size_t bytes() const { return top + (open ? align256(used + 16) : 0); }
  int commit(DevBuf& buf, cudaStream_t s);
};
// A picture as one entry: plane k at pic_planes' offset, copied from src[k] when src is given, device scratch otherwise; no entry space when !on.
template <class V> void stage_picture(Staging& st, V** p, const int16_t* const* src, const b200_geom& g, bool on = true)
{
  for (int k = 0; k < 3; k++) st.put(&p[k], src && k < (g.chromaFormat ? 3 : 1) ? src[k] : nullptr, plane_bytes(g, k), on ? plane_span(g, k) : 0, k == 0);
}
inline void stage_picture(Staging& st, DevPlanes& d, const int16_t* const* src, const b200_geom& g, bool on = true)
{
  for (int k = 0; k < 3; k++) d.stride[k] = g.stride[k];
  stage_picture(st, d.p, src, g, on);
}

// ---- kernel launchers (device pointers, stream-ordered) ----
// Launch hook of a picture context (picture.cu).  A launcher counts each kernel it issues, next to its launch, and brackets its own kernel family with
// begin / end (an event pair when the context profiles).  The kernel-level wrappers (api.cu) pass none.
struct KHook {
  long long launches = 0;
  virtual void begin(int family, cudaStream_t s) = 0;
  virtual void end(int family, cudaStream_t s) = 0;
  virtual ~KHook() {}
};
inline void hook_count(KHook* h) { if (h) h->launches++; }
inline void hook_begin(KHook* h, int family, cudaStream_t s) { if (h) h->begin(family, s); }
inline void hook_end(KHook* h, int family, cudaStream_t s) { if (h) h->end(family, s); }

// Fork/join helper: independent kernels of one stage are spread over auxiliary streams so that their tails overlap.
struct StreamSet {
  cudaStream_t main = nullptr; cudaStream_t aux[4] = {nullptr, nullptr, nullptr, nullptr}; int nAux = 0;
  cudaEvent_t forkEv = nullptr, joinEv[4] = {nullptr, nullptr, nullptr, nullptr};
  bool used[4] = {false, false, false, false};
  StreamSet() {}
  explicit StreamSet(cudaStream_t s) : main(s) {}
  cudaStream_t pick(int i) {            // stream for the i-th independent kernel of the current stage
    if (nAux == 0) return main;
    const int k = i % (nAux + 1);
    if (k == nAux) return main;
    if (!used[k]) { cudaEventRecord(forkEv, main); cudaStreamWaitEvent(aux[k], forkEv, 0); used[k] = true; }
    return aux[k];
  }
  void join() { for (int k = 0; k < nAux; k++) if (used[k]) { cudaEventRecord(joinEv[k], aux[k]); cudaStreamWaitEvent(main, joinEv[k], 0); used[k] = false; } }
};

// ---- device work lists (bucket.cu): index lists + a small block of ints ("meta") per array ----
constexpr int MC_LISTS = 17;     // mode*4 + size class (mode 0 uni, 1 bi, 2 bi+BDOF, 3 DMVR; 32/64/128/256 samples), 16 = affine tiles
constexpr int K1_LISTS = 4;      // TU max dimension <= 8, 16, 32, 64
constexpr int LM_CNT = 0, LM_OFF = 32, LM_CUR = 64, LM_DONE = 96, LM_ERR = 97, LM_INTS = 128;   // meta layout: counts, offsets, cursors, ticket, error bits
int launch_mc_bucket(const b200_pu* pus, size_t numPus, uint32_t* tiles, size_t capTiles, int* meta, const b200_geom& g, int numSlots, int numWp, size_t numDmvr, cudaStream_t s, KHook* hook = nullptr);
int launch_tu_bucket(const b200_tu* tus, size_t numTus, uint32_t* idx, int* meta, const b200_geom& g, size_t numCoefs, size_t numScaling, cudaStream_t s, KHook* hook = nullptr);
int launch_ctu_validate(const b200_sao_ctu* sao, const b200_alf_ctu* alf, const uint8_t* ctuSlice, int nCtu, const CtuLimits& lim, int* meta, cudaStream_t s, KHook* hook);   // after launch_mc_bucket (same meta block)
size_t mc_tile_capacity(const b200_geom& g, size_t numPus);
int num_sms();                   // SM count of the current device (persistent-style grids are sized from it)
int fetch_list_meta(const int* metaDev, int* cnt, int nLists, const char* what, cudaStream_t s);   // synchronises s: list lengths to the host, error bits -> B200_ERR_PARAM

struct K1Launch {
  b200_geom      geom;
  DevPlanes      planes;
  const b200_tu* tus;        // device, caller order
  size_t         numTus;
  const uint32_t* idx;       // device: TU indices bucketed by size class (launch_tu_bucket)
  const int*     meta;       // device: counts / offsets of the 4 lists
  int            cnt[K1_LISTS];   // the same counts on the host (read back after bucketing): exact grids, empty lists are not launched
  const int16_t* coefs;
  const int32_t* scaling;
  int            mode;    // 0: reco = clip(pred + resi); 1: store residual
  int            compSel = 0;             // 0 all TUs, 1 luma TUs only, 2 chroma TUs only (LMCS chroma scaling needs luma first)
  const int*     vpduScale = nullptr;     // device: LMCS chroma residual scale per VPDU, or null
  int16_t*       resi[3] = {nullptr, nullptr, nullptr};   // residual planes (same strides) for TUs flagged B200_TU_RESI, or null: the flag is ignored
};
int launch_k1_residual(const K1Launch& L, StreamSet& ss, KHook* hook = nullptr);

struct LfSliceTab { b200_lf_slice s[64]; };
struct LfLaunch {
  b200_geom geom; DevPlanes planes;
  const b200_lf_param *lfV, *lfH;   // device, [H4][W4] rasters
  const uint8_t* ctuSlice;          // device or null
  LfSliceTab slices; b200_lf_seq seq; int dirs;
};
int launch_lf_deblock(const LfLaunch& L, cudaStream_t s, KHook* hook = nullptr);

// B200_PIC_DERIVE_LF (lf_derive.cu): the edge grids lfV / lfH from CU / TU records; map[2] and mi are [H/4][W/4] scratch (CU maps, LfMi motion field)
struct LfMi;
struct LfDeriveLaunch {
  b200_geom geom;
  const b200_lf_cu* cus; size_t numCus; const b200_lf_tu* tus; const uint32_t* ctuCus; const b200_pu* pus; size_t numPus;
  const b200_lf_slice* slices; const uint8_t* sliceB;
  uint32_t* map[2]; LfMi* mi; b200_lf_param *lfV, *lfH;
  bool anyDisabled;                 // some slice has deblocking disabled
};
constexpr int LM_ERR_LF_RECORD = 32;   // error bit of the PU meta block: a CU / TU record of B200_PIC_DERIVE_LF (lf_cu_problem)
int launch_lf_validate(const b200_lf_cu* cus, size_t numCus, const b200_lf_tu* tus, size_t numTus, const uint32_t* ctuCus, const b200_geom& g, int numSlices, int* meta, cudaStream_t s, KHook* hook);
int launch_lf_derive(const LfDeriveLaunch& L, cudaStream_t s, KHook* hook);

struct SaoLaunch { b200_geom geom; DevPlanes src, dst; const b200_sao_ctu* ctus; b200_vb vb; };
int launch_sao(const SaoLaunch& L, cudaStream_t s, KHook* hook = nullptr);

struct AlfLaunch {
  b200_geom geom; DevPlanes src, dst; const b200_alf_ctu* ctus;
  const int16_t *lumaCoeff, *lumaClip, *chromaCoeff, *chromaClip, *cc[2];
};
int launch_alf(const AlfLaunch& L, StreamSet& ss, KHook* hook = nullptr);   // luma on ss.main, chroma (independent) on an auxiliary stream

constexpr int B200_MAX_SLOTS = 32;
struct McLaunch {
  b200_geom geom; DevPlanes dst;
  const int16_t* refs[B200_MAX_SLOTS * 3] = {};   // device plane pointers per DPB slot
  int refStride[3];
  const b200_pu* pus;               // device
  const uint32_t* tiles;            // device: tile = (puIdx<<6)|(ty<<3)|tx, bucketed into MC_LISTS lists (launch_mc_bucket)
  const int* meta;                  // device: counts / offsets of the lists
  int cnt[MC_LISTS];                // the same counts on the host (read back after bucketing): exact grids, empty lists are not launched
  int32_t* dmvrMv;                  // device or null
  const b200_wp* wp = nullptr;      // device: explicit weighted prediction entries, or null
  const b200_lmcs* lmcs = nullptr;  // device copy of the LMCS tables: luma predictions are stored forward-mapped; null = LMCS off
};
int launch_mc(const McLaunch& L, StreamSet& ss, KHook* hook = nullptr);

struct LmcsLaunch { b200_geom geom; DevPlanes planes; const b200_lmcs* lmcs; const b200_lmcs_vpdu* vpdus; const int16_t* invLut; int* scale; };
int launch_lmcs_vpdu(const LmcsLaunch& L, cudaStream_t s, KHook* hook);   // per-VPDU chroma residual scale from the reconstructed (mapped) luma
int launch_lmcs_inv(const LmcsLaunch& L, cudaStream_t s, KHook* hook);   // inverse map of the luma plane, in place
int launch_lmcs_validate(const b200_lmcs_vpdu* vpdus, const b200_geom& g, int* meta, cudaStream_t s, KHook* hook);   // after launch_mc_bucket (same meta block)

int launch_pack(const DevPlanes& src, const b200_geom& g, int fmt, uint8_t* const dst[3], cudaStream_t s, KHook* hook);   // output.cu: pyuv / 8-bit conversion

// K6 (k6_intra.cu): blocks in decoding order; sync = numTus + 2 ints (done flags, ticket, error bit); owner[c] = one int per 4x4 luma / 2x2 chroma unit
struct IntraLaunch { b200_geom geom; DevPlanes planes; const int16_t* resi[3]; const b200_intra_tu* tus; size_t numTus; int* owner[3]; int ownerStride[3]; size_t ownerBytes[3]; int* sync;
                     int* order = nullptr;      // order: numTus + 8 + 3 * numCtus ints of scratch for the wavefront processing order, or null: list order
                     int compSel = 0;           // 0: every block; 1: luma blocks only; 2: chroma blocks only, continuing a compSel == 1 launch on the same list (LMCS:
                                                // the chroma residual scale of a VPDU is derived from the finished luma, so luma goes first)
                   };
inline size_t intra_order_ints(const b200_geom& g, size_t numTus) { return numTus + 8 + 3 * (size_t)((g.width + g.ctuSize - 1) / g.ctuSize) * ((g.height + g.ctuSize - 1) / g.ctuSize); }
// The owner-map geometry of L's planes (none past the geometry's planes); the maps themselves are the caller's to place
inline void intra_owner_maps(IntraLaunch& L)
{
  const b200_geom& g = L.geom;
  for (int k = 0; k < 3; k++) {
    const int pw = k ? g.width >> 1 : g.width, ph = k ? g.height >> 1 : g.height, unit = k ? 2 : 4;
    L.owner[k] = nullptr; L.ownerStride[k] = k < (g.chromaFormat ? 3 : 1) ? (pw + unit - 1) / unit : 0;
    L.ownerBytes[k] = (size_t)L.ownerStride[k] * ((ph + unit - 1) / unit) * sizeof(int);
  }
}
// The deblocking slice table and sequence parameters (seq null: all zero)
inline void lf_tables(LfLaunch& L, const b200_lf_slice* slices, int numSlices, const b200_lf_seq* seq)
{
  memset(&L.slices, 0, sizeof(L.slices)); memcpy(L.slices.s, slices, numSlices * sizeof(b200_lf_slice));
  if (seq) L.seq = *seq; else memset(&L.seq, 0, sizeof(L.seq));
}
// The ALF tables as one entry: luma coefficients and clips, chroma coefficients and clips, CC-ALF Cb and Cr, back to back (T null: an empty entry)
inline void stage_alf_tables(Staging& st, AlfLaunch& L, const b200_alf_tables* T)
{
  const size_t nL = T ? (size_t)T->numLumaSets * 1300 : 0, nC = T ? (size_t)T->numChromaAlts * 7 : 0, n0 = T ? (size_t)T->numCc[0] * 7 : 0, n1 = T ? (size_t)T->numCc[1] * 7 : 0;
  st.add(&L.lumaCoeff, T ? T->lumaCoeff : nullptr, nL); st.pack(&L.lumaClip, T ? T->lumaClip : nullptr, nL);
  st.pack(&L.chromaCoeff, T ? T->chromaCoeff : nullptr, nC); st.pack(&L.chromaClip, T ? T->chromaClip : nullptr, nC);
  st.pack(&L.cc[0], T ? T->ccCoeff[0] : nullptr, n0); st.pack(&L.cc[1], T ? T->ccCoeff[1] : nullptr, n1);
}
int launch_intra(const IntraLaunch& L, cudaStream_t s, KHook* hook = nullptr);
int launch_intra_ciip_clear(const b200_intra_tu* tus, size_t numTus, int16_t* const resi[3], const int stride[3], cudaStream_t s, KHook* hook);   // before K1: see k6_intra.cu
int launch_intra_validate(const b200_intra_tu* tus, size_t numTus, const b200_geom& g, int* meta, cudaStream_t s, KHook* hook);   // error bit 8 of the PU meta block (after launch_mc_bucket)
// K6 error word (sync[numTus + 1]): bit 1 a wait timed out, bit 2 the blocks of a CTU are not contiguous in the list, bit 4 a CTU holds more blocks than the
// CTU-resident kernel has done bytes for (V2_FLAGS = 3072; only that kernel checks it, and it runs nothing when bit 2 or 4 is set)
constexpr int INTRA_ERR_ORDER = 2, INTRA_ERR_CTU_BLOCKS = 4, INTRA_MAX_CTU_BLOCKS = 3072;
int launch_film_grain(const DevPlanes& src, const DevPlanes& dst, const b200_geom& g, const int8_t* pattern, const uint8_t* sLUT, const uint8_t* pLUT,
                      const uint32_t* lineSeeds, uint32_t* seeds, int scaleShift, const uint8_t present[3], cudaStream_t s, KHook* hook);   // film_grain.cu
int launch_hash(const DevPlanes& src, const b200_geom& g, int method, uint32_t* acc, uint8_t* digest, cudaStream_t s, KHook* hook);   // hash.cu: CRC / checksum of the planes

int ensure_device();   // selects device 0 if none current; fails loudly when there is no sm_90 GPU

}  // namespace b200
