// api.cu — C-ABI entry points of libvvdec_b200.so (include/vvdec_b200.h). Host-pointer wrappers stage
// through device scratch buffers; picture-level entry points keep everything resident (see picture.cu).
#include "common.cuh"
#include "lf_derive.cuh"
#include <stdarg.h>
#include <string.h>
#include <mutex>

namespace b200 {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...)
{
  va_list ap; va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int ensure_device()
{
  static std::once_flag once;
  static int status = 0;
  std::call_once(once, [] {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { set_error("no CUDA device: vvdec_b200 has no CPU fallback"); status = B200_ERR_NO_DEVICE; return; }
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceProp p; cudaGetDeviceProperties(&p, dev);
    if (p.major != 9 || p.minor != 0) { set_error("device %s is sm_%d%d; this library is built for sm_90a only", p.name, p.major, p.minor); status = B200_ERR_NO_DEVICE; }
  });
  if (status) set_error("no usable sm_90 device: vvdec_b200 has no CPU fallback");
  return status;
}

// scratch for the kernel-level host wrappers (single-threaded use, like the reference's per-thread objects): one buffer, laid out per call by a Staging plan
struct HostWrapScratch {
  DevBuf buf;
  cudaStream_t stream = nullptr;
  int init() { if (!stream) { B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)); } return 0; }
};
static HostWrapScratch g_hw;
HostWrapScratch& host_scratch() { return g_hw; }

// whole planes (strides, padding included) of dp back to the caller's planes
static int download_planes(const b200_geom* g, int16_t* const planes[3], const DevPlanes& dp, cudaStream_t s)
{
  for (int c = 0; c < (g->chromaFormat ? 3 : 1); c++) B200_CUDA(cudaMemcpyAsync(planes[c], dp.p[c], plane_bytes(*g, c), cudaMemcpyDeviceToHost, s));
  return 0;
}

int num_sms()
{
  static int cache[64] = {0};
  int dev = 0; cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!cache[dev]) { int n = 0; if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132; cache[dev] = n; }
  return cache[dev];
}

// waits for a bucketing pass, copies its list lengths to the host and turns its error bits into B200_ERR_PARAM
int fetch_list_meta(const int* metaDev, int* cnt, int nLists, const char* what, cudaStream_t s)
{
  int h[LM_INTS];
  B200_CUDA(cudaMemcpyAsync(h, metaDev, sizeof(h), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  for (int i = 0; i < nLists; i++) cnt[i] = h[LM_CNT + i];
  B200_CHECK(!(h[LM_ERR] & 1), "%s: invalid record (reference slots, block size or flag combination)", what);
  B200_CHECK(!(h[LM_ERR] & 2), "%s: more tiles than the picture can hold (overlapping PUs?)", what);
  return 0;
}

// The host half of the rules (rules.cuh): false, with the error set to the entry point's name and the reason, when `why` is a reason.
static bool rule_ok(const char* fn, const char* why)
{
  if (why) set_error("%s: %s", fn, why);
  return !why;
}
// every record of a list: problem(i) is the reason record i is refused, or null
template <class F> static bool records_ok(const char* fn, const char* what, size_t n, F problem)
{
  for (size_t i = 0; i < n; i++)
    if (const char* why = problem(i)) { set_error("%s: %s %zu: %s", fn, what, i, why); return false; }
  return true;
}

}  // namespace b200

using namespace b200;

extern "C" {

B200_API const char* b200_last_error(void) { return g_err; }
B200_API const char* b200_version(void) { return "vvdec_b200 0.1 (sm_90a)"; }
B200_API int b200_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }

B200_API int b200_k1_residual(const b200_geom* g, int16_t* const planes[3], const b200_tu* tus, size_t numTus,
                              const int16_t* coefs, size_t numCoefs, const int32_t* scaling, size_t numScaling, int mode)
{
  B200_CHECK(g && planes && (tus || !numTus), "b200_k1_residual: null argument");
  const TuLimits lim = tu_limits(*g, numCoefs, numScaling);
  if (!rule_ok("b200_k1_residual", geom_problem(*g, 12, 1)) || !records_ok("b200_k1_residual", "TU record", numTus, [&](size_t i) { return tu_problem(tus[i], lim); }))
    return B200_ERR_PARAM;
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  K1Launch L; L.geom = *g; L.numTus = numTus; L.mode = mode;
  int* meta; uint32_t* idx;
  Staging st;
  stage_picture(st, L.planes, planes, *g); st.add(&L.tus, tus, numTus); st.add(&L.coefs, coefs, numCoefs); st.add(&L.scaling, scaling, numScaling);
  st.add(&meta, nullptr, LM_INTS); st.add(&idx, nullptr, numTus);
  if (int rc = st.commit(g_hw.buf, s)) return rc;
  if (int rc = launch_tu_bucket(L.tus, numTus, idx, meta, *g, numCoefs, numScaling, s)) return rc;
  L.idx = idx; L.meta = meta;
  if (int rc = fetch_list_meta(meta, L.cnt, K1_LISTS, "b200_k1_residual", s)) return rc;
  StreamSet ss(s);
  if (int rc = launch_k1_residual(L, ss)) return rc;
  if (int rc = download_planes(g, planes, L.planes, s)) return rc;
  B200_CUDA(cudaStreamSynchronize(s));
  return 0;
}

B200_API int b200_lf_deblock(const b200_geom* g, int16_t* const planes[3], const b200_lf_param* lfV, const b200_lf_param* lfH,
                             const uint8_t* ctuSlice, const b200_lf_slice* slices, int numSlices, const b200_lf_seq* seq, int dirs)
{
  B200_CHECK(g && planes && lfV && lfH && slices, "b200_lf_deblock: null argument");
  B200_CHECK(numSlices >= 1 && numSlices <= 64, "b200_lf_deblock: numSlices %d out of range 1..64", numSlices);
  if (!rule_ok("b200_lf_deblock", geom_problem(*g, 12, 1))) return B200_ERR_PARAM;
  B200_CHECK(!(dirs & ~3), "b200_lf_deblock: dirs %d (bit 0 vertical, bit 1 horizontal edges)", dirs);
  B200_CHECK(!seq || !seq->ladfEnabled || (seq->ladfNumIntervals >= 2 && seq->ladfNumIntervals <= 5), "b200_lf_deblock: %d LADF intervals (2..5)", seq ? seq->ladfNumIntervals : 0);
  const size_t n4 = (size_t)((g->width + 3) >> 2) * ((g->height + 3) >> 2);
  const size_t nCtu = (size_t)((g->width + g->ctuSize - 1) / g->ctuSize) * ((g->height + g->ctuSize - 1) / g->ctuSize);
  for (size_t i = 0; ctuSlice && i < nCtu; i++) B200_CHECK(ctuSlice[i] < numSlices, "b200_lf_deblock: CTU %zu is in slice %d of %d", i, ctuSlice[i], numSlices);
  for (int dir = 0; dir < 2; dir++) {
    int x = 0, y = 0;
    if (const char* why = lf_grid_problem(*g, dir ? lfH : lfV, dir, &x, &y)) { set_error("b200_lf_deblock: %s edge at (%d, %d): %s", dir ? "lfH" : "lfV", x, y, why); return B200_ERR_PARAM; }
  }
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  LfLaunch L; L.geom = *g; L.dirs = dirs;
  lf_tables(L, slices, numSlices, seq);
  Staging st;
  stage_picture(st, L.planes, planes, *g); st.add(&L.lfV, lfV, n4); st.add(&L.lfH, lfH, n4); st.add(&L.ctuSlice, ctuSlice, ctuSlice ? nCtu : 0);
  if (int rc = st.commit(g_hw.buf, s)) return rc;
  if (int rc = launch_lf_deblock(L, s)) return rc;
  if (int rc = download_planes(g, planes, L.planes, s)) return rc;
  B200_CUDA(cudaStreamSynchronize(s));
  return 0;
}

B200_API int b200_lf_derive(const b200_geom* g, const b200_lf_cu* cus, size_t numCus, const b200_lf_tu* tus, size_t numTus, const uint32_t* ctuCus,
                            const b200_pu* pus, size_t numPus, const b200_lf_slice* slices, const uint8_t* sliceB, int numSlices, b200_lf_param* lfV, b200_lf_param* lfH)
{
  const char* fn = "b200_lf_derive";
  B200_CHECK(g && cus && numCus && tus && ctuCus && (pus || !numPus) && slices && sliceB && lfV && lfH, "b200_lf_derive: null argument");
  B200_CHECK(numSlices >= 1 && numSlices <= 64, "b200_lf_derive: numSlices %d out of range 1..64", numSlices);
  if (!rule_ok(fn, geom_problem(*g, 12, 1))) return B200_ERR_PARAM;
  const size_t n4 = (size_t)(g->width >> 2) * (g->height >> 2);
  const int nCtu = ((g->width + g->ctuSize - 1) / g->ctuSize) * ((g->height + g->ctuSize - 1) / g->ctuSize);
  B200_CHECK(ctuCus[0] == 0 && ctuCus[nCtu] == numCus, "b200_lf_derive: the CTU ranges do not cover the CU records from 0 to numCus");
  const LfLimits lim = lf_limits(*g, numSlices, numTus);
  for (int a = 0; a < nCtu; a++) {
    B200_CHECK(ctuCus[a] <= ctuCus[a + 1], "b200_lf_derive: the CU range of CTU %d ends before it starts", a);
    for (uint32_t i = ctuCus[a]; i < ctuCus[a + 1]; i++)
      if (const char* why = lf_cu_problem(cus[i], tus, a, lim)) { set_error("b200_lf_derive: CU record %u of CTU %d: %s", i, a, why); return B200_ERR_PARAM; }
  }
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  LfDeriveLaunch L{}; L.geom = *g; L.numCus = numCus; L.numPus = numPus;
  Staging st;
  st.add(&L.cus, cus, numCus); st.add(&L.tus, tus, numTus); st.add(&L.ctuCus, ctuCus, (size_t)nCtu + 1); st.add(&L.pus, pus, numPus);
  st.add(&L.slices, slices, (size_t)numSlices); st.add(&L.sliceB, sliceB, (size_t)numSlices);
  st.add(&L.map[0], nullptr, 2 * n4); st.add(&L.mi, nullptr, n4); st.add(&L.lfV, nullptr, n4); st.add(&L.lfH, nullptr, n4);
  if (int rc = st.commit(g_hw.buf, s)) return rc;
  L.map[1] = L.map[0] + n4;
  L.anyDisabled = false;
  for (int k = 0; k < numSlices; k++) L.anyDisabled = L.anyDisabled || slices[k].disable;
  if (int rc = launch_lf_derive(L, s, nullptr)) return rc;
  if (int rc = copy_host(lfV, L.lfV, n4 * sizeof(b200_lf_param), cudaMemcpyDeviceToHost, s)) return rc;
  if (int rc = copy_host(lfH, L.lfH, n4 * sizeof(b200_lf_param), cudaMemcpyDeviceToHost, s)) return rc;
  B200_CUDA(cudaStreamSynchronize(s));
  return 0;
}

// dst planes of the kernel-level filters: only the plane width of each row goes back, so the caller's stride padding keeps what it held
static int download_plane_rows(const b200_geom* g, int16_t* const planes[3], const DevPlanes& dp, cudaStream_t s)
{
  for (int c = 0; c < (g->chromaFormat ? 3 : 1); c++) {
    const size_t pitch = (size_t)g->stride[c] * sizeof(int16_t);
    B200_CUDA(cudaMemcpy2DAsync(planes[c], pitch, dp.p[c], pitch, (size_t)(c ? g->width >> 1 : g->width) * sizeof(int16_t), c ? g->height >> 1 : g->height, cudaMemcpyDeviceToHost, s));
  }
  return 0;
}

B200_API int b200_sao_picture(const b200_geom* g, const int16_t* const src[3], int16_t* const dst[3], const b200_sao_ctu* ctus, const b200_vb* vb)
{
  B200_CHECK(g && src && dst && ctus, "b200_sao_picture: null argument");
  const char* fn = "b200_sao_picture";
  if (!rule_ok(fn, geom_problem(*g, 12, 4)) || (vb && !rule_ok(fn, vb_problem(*vb, g->width, g->height)))) return B200_ERR_PARAM;
  const CtuLimits cl = ctu_limits(*g, nullptr, 0);
  if (!records_ok(fn, "CTU", (size_t)cl.ctusW * cl.ctusH, [&](size_t i) { return sao_ctu_problem(ctus[i], g->chromaFormat ? 3 : 1); })) return B200_ERR_PARAM;
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  SaoLaunch L; L.geom = *g;
  if (vb) L.vb = *vb; else memset(&L.vb, 0, sizeof(L.vb));
  Staging st;
  stage_picture(st, L.src, src, *g); stage_picture(st, L.dst, nullptr, *g); st.add(&L.ctus, ctus, (size_t)cl.ctusW * cl.ctusH);
  if (int rc = st.commit(g_hw.buf, s)) return rc;
  if (int rc = launch_sao(L, s)) return rc;
  if (int rc = download_plane_rows(g, dst, L.dst, s)) return rc;
  B200_CUDA(cudaStreamSynchronize(s));
  return 0;
}

B200_API int b200_intra_reconstruct(const b200_geom* g, int16_t* const planes[3], const int16_t* const resi[3], const b200_intra_tu* tus, size_t numTus)
{
  B200_CHECK(g && planes && (tus || !numTus), "b200_intra_reconstruct: null argument");
  const int nPl = g->chromaFormat ? 3 : 1;
  if (!rule_ok("b200_intra_reconstruct", geom_problem(*g, 12, 1))
      || !records_ok("b200_intra_reconstruct", "intra block record", numTus, [&](size_t i) { return intra_problem(tus[i], i ? &tus[i - 1] : nullptr, *g); }))
    return B200_ERR_PARAM;
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  IntraLaunch L; L.geom = *g; L.numTus = numTus;
  intra_owner_maps(L);
  Staging st;
  stage_picture(st, L.planes, planes, *g);
  for (int c = 0; c < 3; c++) st.add(&L.resi[c], resi ? resi[c] : nullptr, c < nPl && resi && resi[c] ? plane_bytes(*g, c) / 2 : 0);
  for (int c = 0; c < nPl; c++) st.add(&L.owner[c], nullptr, L.ownerBytes[c] / sizeof(int));
  st.add(&L.tus, tus, numTus); st.add(&L.sync, nullptr, numTus + 2); st.add(&L.order, nullptr, intra_order_ints(*g, numTus));
  if (int rc = st.commit(g_hw.buf, s)) return rc;
  if (int rc = launch_intra(L, s)) return rc;
  int err = 0;
  if (numTus) B200_CUDA(cudaMemcpyAsync(&err, L.sync + numTus + 1, sizeof(int), cudaMemcpyDeviceToHost, s));
  if (int rc = download_planes(g, planes, L.planes, s)) return rc;
  B200_CUDA(cudaStreamSynchronize(s));
  B200_CHECK(!(err & INTRA_ERR_CTU_BLOCKS), "b200_intra_reconstruct: a CTU holds more than %d intra block records (overlapping records?)", INTRA_MAX_CTU_BLOCKS);
  B200_CHECK(!err, "b200_intra_reconstruct: a block waited for a neighbour that never finished, or the blocks of a CTU are not contiguous (list not in decoding order?)");
  return 0;
}

B200_API int b200_intra_predict(const b200_geom* g, int16_t* const planes[3], const b200_intra_tu* tus, size_t numTus)
{
  return b200_intra_reconstruct(g, planes, nullptr, tus, numTus);
}

B200_API int b200_alf_picture(const b200_geom* g, const int16_t* const src[3], int16_t* const dst[3], const b200_alf_ctu* ctus, const b200_alf_tables* T)
{
  B200_CHECK(g && src && dst && ctus && T, "b200_alf_picture: null argument");
  // ALF is defined up to 10 bit (the reference's AdaptiveLoopFilter::create refuses more, and its clipping values exist for 8, 9 and 10 bit only)
  const char* fn = "b200_alf_picture";
  if (!rule_ok(fn, geom_problem(*g, 10, 4)) || !rule_ok(fn, alf_tables_problem(*T, 24))) return B200_ERR_PARAM;
  const CtuLimits cl = ctu_limits(*g, T, 0);
  if (!records_ok(fn, "CTU", (size_t)cl.ctusW * cl.ctusH, [&](size_t i) { return alf_ctu_problem(ctus[i], (int)i, cl); })) return B200_ERR_PARAM;
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  AlfLaunch L; L.geom = *g;
  Staging st;
  stage_picture(st, L.src, src, *g); stage_picture(st, L.dst, nullptr, *g); st.add(&L.ctus, ctus, (size_t)cl.ctusW * cl.ctusH); stage_alf_tables(st, L, T);
  if (int rc = st.commit(g_hw.buf, s)) return rc;
  StreamSet ss(s);
  if (int rc = launch_alf(L, ss)) return rc;
  if (int rc = download_plane_rows(g, dst, L.dst, s)) return rc;
  B200_CUDA(cudaStreamSynchronize(s));
  return 0;
}

B200_API int b200_mc_predict(const b200_geom* g, int16_t* const dst[3], const int16_t* const* refs, int numSlots,
                             const b200_pu* pus, size_t numPus, int32_t* dmvrMv, size_t numDmvr)
{
  return b200_mc_predict_wp(g, dst, refs, numSlots, pus, numPus, dmvrMv, numDmvr, nullptr, 0);
}

B200_API int b200_mc_predict_wp(const b200_geom* g, int16_t* const dst[3], const int16_t* const* refs, int numSlots,
                                const b200_pu* pus, size_t numPus, int32_t* dmvrMv, size_t numDmvr, const b200_wp* wp, int numWp)
{
  B200_CHECK(g && dst && refs && (pus || !numPus), "b200_mc_predict: null argument");
  if (!rule_ok("b200_mc_predict", geom_problem(*g, 12, 1))) return B200_ERR_PARAM;
  B200_CHECK(numSlots >= 1 && numSlots <= B200_MAX_SLOTS, "b200_mc_predict: numSlots %d", numSlots);
  B200_CHECK(numPus < (1u << 26), "b200_mc_predict: too many PUs");
  B200_CHECK(!wp || numWp <= 255, "b200_mc_predict_wp: at most 255 weighted-prediction entries");
  const PuLimits lim = pu_limits(*g, numSlots, wp ? numWp : 0, numDmvr);
  if (!records_ok("b200_mc_predict", "PU", numPus, [&](size_t i) { return pu_problem(pus[i], lim); })) return B200_ERR_PARAM;
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  McLaunch L; L.geom = *g;
  const size_t capTiles = mc_tile_capacity(*g, numPus);
  int* meta; uint32_t* tiles;
  Staging st;
  stage_picture(st, L.dst, dst, *g);
  for (int sl = 0; sl < numSlots; sl++) stage_picture(st, &L.refs[sl * 3], &refs[sl * 3], *g);
  st.add(&L.pus, pus, numPus); st.add(&meta, nullptr, LM_INTS); st.add(&tiles, nullptr, capTiles); st.add(&L.dmvrMv, nullptr, dmvrMv ? numDmvr * 2 : 0);
  st.add(&L.wp, wp, wp && numWp > 0 ? numWp : 0);
  if (int rc = st.commit(g_hw.buf, s)) return rc;
  for (int c = 0; c < 3; c++) L.refStride[c] = g->stride[c];
  if (int rc = launch_mc_bucket(L.pus, numPus, tiles, capTiles, meta, *g, numSlots, wp ? numWp : 0, numDmvr, s)) return rc;
  L.tiles = tiles; L.meta = meta;
  if (int rc = fetch_list_meta(meta, L.cnt, MC_LISTS, "b200_mc_predict", s)) return rc;
  if (L.dmvrMv) B200_CUDA(cudaMemsetAsync(L.dmvrMv, 0, numDmvr * 8, s));
  StreamSet ss(s);
  if (int rc = launch_mc(L, ss)) return rc;
  if (int rc = download_planes(g, dst, L.dst, s)) return rc;
  if (L.dmvrMv) B200_CUDA(cudaMemcpyAsync(dmvrMv, L.dmvrMv, numDmvr * 8, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
