// common.cuh — shared device/host helpers for the sm_90a kernels of vvdec_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
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

// ---- kernel launchers (device pointers, stream-ordered) ----
// optional per-family event recorder (picture.cu); launchers call prof->begin(f)/end(f) around their kernels
struct KProf { virtual void begin(int family, cudaStream_t s) = 0; virtual void end(int family, cudaStream_t s) = 0; virtual ~KProf() {} };

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
int launch_mc_bucket(const b200_pu* pus, size_t numPus, uint32_t* tiles, size_t capTiles, int* meta, const b200_geom& g, int numSlots, int numWp, size_t numDmvr, cudaStream_t s);
int launch_tu_bucket(const b200_tu* tus, size_t numTus, uint32_t* idx, int* meta, const b200_geom& g, size_t numCoefs, size_t numScaling, cudaStream_t s);
int launch_ctu_validate(const b200_sao_ctu* sao, const b200_alf_ctu* alf, const uint8_t* ctuSlice, int nCtu, const CtuLimits& lim, int* meta, cudaStream_t s);   // after launch_mc_bucket (same meta block)
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
int launch_k1_residual(const K1Launch& L, StreamSet& ss, KProf* prof = nullptr);

struct LfSliceTab { b200_lf_slice s[64]; };
struct LfLaunch {
  b200_geom geom; DevPlanes planes;
  const b200_lf_param *lfV, *lfH;   // device, [H4][W4] rasters
  const uint8_t* ctuSlice;          // device or null
  LfSliceTab slices; b200_lf_seq seq; int dirs;
};
int launch_lf_deblock(const LfLaunch& L, cudaStream_t s, KProf* prof = nullptr);

struct SaoLaunch { b200_geom geom; DevPlanes src, dst; const b200_sao_ctu* ctus; b200_vb vb; };
int launch_sao(const SaoLaunch& L, cudaStream_t s, KProf* prof = nullptr);

struct AlfLaunch {
  b200_geom geom; DevPlanes src, dst; const b200_alf_ctu* ctus;
  const int16_t *lumaCoeff, *lumaClip, *chromaCoeff, *chromaClip, *cc[2];
};
int launch_alf(const AlfLaunch& L, StreamSet& ss, KProf* prof = nullptr);   // luma on ss.main, chroma (independent) on an auxiliary stream

constexpr int B200_MAX_SLOTS = 32;
struct McLaunch {
  b200_geom geom; DevPlanes dst;
  const int16_t* refs[B200_MAX_SLOTS * 3];   // device plane pointers per DPB slot
  int refStride[3];
  const b200_pu* pus;               // device
  const uint32_t* tiles;            // device: tile = (puIdx<<6)|(ty<<3)|tx, bucketed into MC_LISTS lists (launch_mc_bucket)
  const int* meta;                  // device: counts / offsets of the lists
  int cnt[MC_LISTS];                // the same counts on the host (read back after bucketing): exact grids, empty lists are not launched
  int32_t* dmvrMv;                  // device or null
  const b200_wp* wp = nullptr;      // device: explicit weighted prediction entries, or null
  const b200_lmcs* lmcs = nullptr;  // device copy of the LMCS tables: luma predictions are stored forward-mapped; null = LMCS off
};
int launch_mc(const McLaunch& L, StreamSet& ss, KProf* prof = nullptr);
int mc_launch_count(const McLaunch& L);
int k1_launch_count(const K1Launch& L);

struct LmcsLaunch { b200_geom geom; DevPlanes planes; const b200_lmcs* lmcs; const b200_lmcs_vpdu* vpdus; const int16_t* invLut; int* scale; };
int launch_lmcs_vpdu(const LmcsLaunch& L, cudaStream_t s);   // per-VPDU chroma residual scale from the reconstructed (mapped) luma
int launch_lmcs_inv(const LmcsLaunch& L, cudaStream_t s);    // inverse map of the luma plane, in place
int launch_lmcs_validate(const b200_lmcs_vpdu* vpdus, const b200_geom& g, int* meta, cudaStream_t s);   // after launch_mc_bucket (same meta block)

int launch_pack(const DevPlanes& src, const b200_geom& g, int fmt, uint8_t* const dst[3], cudaStream_t s);   // output.cu: pyuv / 8-bit conversion

// K6 (k6_intra.cu): blocks in decoding order; sync = numTus + 2 ints (done flags, ticket, error bit); owner[c] = one int per 4x4 luma / 2x2 chroma unit
struct IntraLaunch { b200_geom geom; DevPlanes planes; const int16_t* resi[3]; const b200_intra_tu* tus; size_t numTus; int* owner[3]; int ownerStride[3]; size_t ownerBytes[3]; int* sync;
                     int* order = nullptr;      // order: numTus + 8 + 3 * numCtus ints of scratch for the wavefront processing order, or null: list order
                     int compSel = 0;           // 0: every block; 1: luma blocks only; 2: chroma blocks only, continuing a compSel == 1 launch on the same list (LMCS:
                                                // the chroma residual scale of a VPDU is derived from the finished luma, so luma goes first)
                   };
inline size_t intra_order_ints(const b200_geom& g, size_t numTus) { return numTus + 8 + 3 * (size_t)((g.width + g.ctuSize - 1) / g.ctuSize) * ((g.height + g.ctuSize - 1) / g.ctuSize); }
int launch_intra(const IntraLaunch& L, cudaStream_t s);
int launch_intra_ciip_clear(const b200_intra_tu* tus, size_t numTus, int16_t* const resi[3], const int stride[3], cudaStream_t s);   // before K1: see k6_intra.cu
int launch_intra_validate(const b200_intra_tu* tus, size_t numTus, const b200_geom& g, int* meta, cudaStream_t s);   // error bit 8 of the PU meta block (after launch_mc_bucket)
// K6 error word (sync[numTus + 1]): bit 1 a wait timed out, bit 2 the blocks of a CTU are not contiguous in the list, bit 4 a CTU holds more blocks than the
// CTU-resident kernel has done bytes for (V2_FLAGS = 3072; only that kernel checks it, and it runs nothing when bit 2 or 4 is set)
constexpr int INTRA_ERR_ORDER = 2, INTRA_ERR_CTU_BLOCKS = 4, INTRA_MAX_CTU_BLOCKS = 3072;
int launch_film_grain(const DevPlanes& src, const DevPlanes& dst, const b200_geom& g, const int8_t* pattern, const uint8_t* sLUT, const uint8_t* pLUT,
                      const uint32_t* lineSeeds, uint32_t* seeds, int scaleShift, const uint8_t present[3], cudaStream_t s);   // film_grain.cu
int launch_hash(const DevPlanes& src, const b200_geom& g, int method, uint32_t* acc, uint8_t* digest, cudaStream_t s);   // hash.cu: CRC / checksum of the planes

int ensure_device();   // selects device 0 if none current; fails loudly when there is no sm_90 GPU

}  // namespace b200
