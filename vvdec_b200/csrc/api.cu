// api.cu — C-ABI entry points of libvvdec_b200.so (include/vvdec_b200.h). Host-pointer wrappers stage
// through device scratch buffers; picture-level entry points keep everything resident (see picture.cu).
#include "common.cuh"
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

// scratch for the kernel-level host wrappers (single-threaded use, like the reference's per-thread objects)
struct HostWrapScratch {
  DevBuf planes[3], tus, coefs, scaling, misc[8];
  cudaStream_t stream = nullptr;
  int init() { if (!stream) { B200_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)); } return 0; }
};
static HostWrapScratch g_hw;
HostWrapScratch& host_scratch() { return g_hw; }

// Upload the three host planes described by g into scratch; fills dp.
static int upload_planes(const b200_geom* g, int16_t* const planes[3], DevPlanes& dp, cudaStream_t s)
{
  const int nPlanes = g->chromaFormat ? 3 : 1;
  for (int c = 0; c < nPlanes; c++) {
    const int ph = c ? g->height >> 1 : g->height;
    const size_t bytes = (size_t)g->stride[c] * ph * sizeof(int16_t);
    if (int rc = g_hw.planes[c].reserve(bytes)) return rc;
    dp.p[c] = g_hw.planes[c].as<int16_t>(); dp.stride[c] = g->stride[c];
    B200_CUDA(cudaMemcpyAsync(dp.p[c], planes[c], bytes, cudaMemcpyHostToDevice, s));
  }
  return 0;
}
static int download_planes(const b200_geom* g, int16_t* const planes[3], const DevPlanes& dp, cudaStream_t s)
{
  const int nPlanes = g->chromaFormat ? 3 : 1;
  for (int c = 0; c < nPlanes; c++) {
    const int ph = c ? g->height >> 1 : g->height;
    B200_CUDA(cudaMemcpyAsync(planes[c], dp.p[c], (size_t)g->stride[c] * ph * sizeof(int16_t), cudaMemcpyDeviceToHost, s));
  }
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
  if (int rc = upload_planes(g, planes, L.planes, s)) return rc;
  if (int rc = g_hw.tus.reserve(numTus * sizeof(b200_tu))) return rc;
  if (int rc = g_hw.coefs.reserve(numCoefs * sizeof(int16_t) + 16)) return rc;
  if (int rc = g_hw.scaling.reserve(numScaling * sizeof(int32_t) + 16)) return rc;
  if (int rc = g_hw.misc[4].reserve(numTus * 4 + LM_INTS * sizeof(int) + 256)) return rc;
  if (numTus) B200_CUDA(cudaMemcpyAsync(g_hw.tus.p, tus, numTus * sizeof(b200_tu), cudaMemcpyHostToDevice, s));
  if (numCoefs) B200_CUDA(cudaMemcpyAsync(g_hw.coefs.p, coefs, numCoefs * sizeof(int16_t), cudaMemcpyHostToDevice, s));
  if (numScaling) B200_CUDA(cudaMemcpyAsync(g_hw.scaling.p, scaling, numScaling * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  L.tus = g_hw.tus.as<b200_tu>(); L.coefs = g_hw.coefs.as<int16_t>(); L.scaling = g_hw.scaling.as<int32_t>();
  int* meta = g_hw.misc[4].as<int>(); uint32_t* idx = reinterpret_cast<uint32_t*>(meta + LM_INTS);
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
  memset(&L.slices, 0, sizeof(L.slices)); memcpy(L.slices.s, slices, numSlices * sizeof(b200_lf_slice));
  if (seq) L.seq = *seq; else memset(&L.seq, 0, sizeof(L.seq));
  if (int rc = upload_planes(g, planes, L.planes, s)) return rc;
  if (int rc = g_hw.misc[0].reserve(n4 * sizeof(b200_lf_param))) return rc;
  if (int rc = g_hw.misc[1].reserve(n4 * sizeof(b200_lf_param))) return rc;
  if (int rc = g_hw.misc[2].reserve(nCtu)) return rc;
  B200_CUDA(cudaMemcpyAsync(g_hw.misc[0].p, lfV, n4 * sizeof(b200_lf_param), cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(g_hw.misc[1].p, lfH, n4 * sizeof(b200_lf_param), cudaMemcpyHostToDevice, s));
  if (ctuSlice) B200_CUDA(cudaMemcpyAsync(g_hw.misc[2].p, ctuSlice, nCtu, cudaMemcpyHostToDevice, s));
  L.lfV = g_hw.misc[0].as<b200_lf_param>(); L.lfH = g_hw.misc[1].as<b200_lf_param>();
  L.ctuSlice = ctuSlice ? g_hw.misc[2].as<uint8_t>() : nullptr;
  if (int rc = launch_lf_deblock(L, s)) return rc;
  if (int rc = download_planes(g, planes, L.planes, s)) return rc;
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

static int upload_src_alloc_dst(const b200_geom* g, const int16_t* const src[3], DevPlanes& ds, DevPlanes& dd, cudaStream_t s)
{
  const int nPlanes = g->chromaFormat ? 3 : 1;
  for (int c = 0; c < nPlanes; c++) {
    const int ph = c ? g->height >> 1 : g->height;
    const size_t bytes = (size_t)g->stride[c] * ph * sizeof(int16_t);
    if (int rc = g_hw.planes[c].reserve(bytes)) return rc;
    if (int rc = g_hw.misc[3 + c].reserve(bytes)) return rc;
    ds.p[c] = g_hw.planes[c].as<int16_t>(); dd.p[c] = g_hw.misc[3 + c].as<int16_t>(); ds.stride[c] = dd.stride[c] = g->stride[c];
    B200_CUDA(cudaMemcpyAsync(ds.p[c], src[c], bytes, cudaMemcpyHostToDevice, s));
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
  if (int rc = upload_src_alloc_dst(g, src, L.src, L.dst, s)) return rc;
  const size_t nCtu = (size_t)cl.ctusW * cl.ctusH;
  if (int rc = g_hw.misc[0].reserve(nCtu * sizeof(b200_sao_ctu))) return rc;
  B200_CUDA(cudaMemcpyAsync(g_hw.misc[0].p, ctus, nCtu * sizeof(b200_sao_ctu), cudaMemcpyHostToDevice, s));
  L.ctus = g_hw.misc[0].as<b200_sao_ctu>();
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
  if (int rc = upload_planes(g, planes, L.planes, s)) return rc;
  for (int c = 0; c < 3; c++) {
    L.resi[c] = nullptr; L.owner[c] = nullptr; L.ownerStride[c] = 0; L.ownerBytes[c] = 0;
    if (c >= nPl) continue;
    const int pw = c ? g->width >> 1 : g->width, ph = c ? g->height >> 1 : g->height, unit = c ? 2 : 4;
    L.ownerStride[c] = (pw + unit - 1) / unit; L.ownerBytes[c] = (size_t)L.ownerStride[c] * ((ph + unit - 1) / unit) * sizeof(int);
    if (int rc = g_hw.misc[c].reserve(L.ownerBytes[c])) return rc;
    L.owner[c] = g_hw.misc[c].as<int>();
    if (resi && resi[c]) {
      const size_t bytes = (size_t)g->stride[c] * ph * sizeof(int16_t);
      if (int rc = g_hw.misc[3 + c].reserve(bytes)) return rc;
      B200_CUDA(cudaMemcpyAsync(g_hw.misc[3 + c].p, resi[c], bytes, cudaMemcpyHostToDevice, s));
      L.resi[c] = g_hw.misc[3 + c].as<int16_t>();
    }
  }
  if (int rc = g_hw.tus.reserve(numTus * sizeof(b200_intra_tu) + 16)) return rc;
  if (int rc = g_hw.misc[6].reserve((numTus + 2) * sizeof(int))) return rc;
  if (int rc = g_hw.misc[7].reserve(intra_order_ints(*g, numTus) * sizeof(int))) return rc;
  if (numTus) B200_CUDA(cudaMemcpyAsync(g_hw.tus.p, tus, numTus * sizeof(b200_intra_tu), cudaMemcpyHostToDevice, s));
  L.tus = g_hw.tus.as<b200_intra_tu>(); L.sync = g_hw.misc[6].as<int>(); L.order = g_hw.misc[7].as<int>();
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
  if (int rc = upload_src_alloc_dst(g, src, L.src, L.dst, s)) return rc;
  const size_t nCtu = (size_t)cl.ctusW * cl.ctusH;
  const size_t nL = (size_t)T->numLumaSets * 1300, nC = (size_t)T->numChromaAlts * 7, n0 = (size_t)T->numCc[0] * 7, n1 = (size_t)T->numCc[1] * 7;
  const size_t tabElems = 2 * nL + 2 * nC + n0 + n1 + 8;
  if (int rc = g_hw.misc[0].reserve(nCtu * sizeof(b200_alf_ctu))) return rc;
  if (int rc = g_hw.misc[1].reserve(tabElems * sizeof(int16_t))) return rc;
  B200_CUDA(cudaMemcpyAsync(g_hw.misc[0].p, ctus, nCtu * sizeof(b200_alf_ctu), cudaMemcpyHostToDevice, s));
  int16_t* d = g_hw.misc[1].as<int16_t>();
  auto up = [&](const int16_t* h, size_t n, const int16_t*& out) -> int {
    out = d; if (n) B200_CUDA(cudaMemcpyAsync(d, h, n * sizeof(int16_t), cudaMemcpyHostToDevice, s)); d += n; return 0; };
  if (int rc = up(T->lumaCoeff, nL, L.lumaCoeff)) return rc;
  if (int rc = up(T->lumaClip, nL, L.lumaClip)) return rc;
  if (int rc = up(T->chromaCoeff, nC, L.chromaCoeff)) return rc;
  if (int rc = up(T->chromaClip, nC, L.chromaClip)) return rc;
  if (int rc = up(T->ccCoeff[0], n0, L.cc[0])) return rc;
  if (int rc = up(T->ccCoeff[1], n1, L.cc[1])) return rc;
  L.ctus = g_hw.misc[0].as<b200_alf_ctu>();
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
  if (int rc = upload_planes(g, dst, L.dst, s)) return rc;
  const int nPlanes = g->chromaFormat ? 3 : 1;
  size_t planeBytes[3] = {0, 0, 0}, total = 0;
  for (int c = 0; c < nPlanes; c++) { planeBytes[c] = (((size_t)g->stride[c] * (c ? g->height >> 1 : g->height) * 2) + 255) & ~(size_t)255; total += planeBytes[c]; }
  if (int rc = g_hw.misc[3].reserve(total * numSlots)) return rc;
  std::vector<const int16_t*> ptrs(numSlots * 3, nullptr);
  char* base = g_hw.misc[3].as<char>();
  for (int sl = 0; sl < numSlots; sl++) {
    size_t off = 0;
    for (int c = 0; c < nPlanes; c++) {
      char* d = base + (size_t)sl * total + off;
      B200_CUDA(cudaMemcpyAsync(d, refs[sl * 3 + c], (size_t)g->stride[c] * (c ? g->height >> 1 : g->height) * 2, cudaMemcpyHostToDevice, s));
      ptrs[sl * 3 + c] = reinterpret_cast<const int16_t*>(d); off += planeBytes[c];
    }
  }
  const size_t capTiles = mc_tile_capacity(*g, numPus);
  if (int rc = g_hw.misc[5].reserve(numPus * sizeof(b200_pu) + 64)) return rc;
  if (int rc = g_hw.misc[6].reserve(capTiles * 4 + LM_INTS * sizeof(int) + 256)) return rc;
  if (int rc = g_hw.misc[7].reserve(numDmvr * 8 + 64)) return rc;
  if (numPus) B200_CUDA(cudaMemcpyAsync(g_hw.misc[5].p, pus, numPus * sizeof(b200_pu), cudaMemcpyHostToDevice, s));
  int* meta = g_hw.misc[6].as<int>(); uint32_t* tiles = reinterpret_cast<uint32_t*>(meta + LM_INTS);
  if (int rc = launch_mc_bucket(g_hw.misc[5].as<b200_pu>(), numPus, tiles, capTiles, meta, *g, numSlots, wp ? numWp : 0, numDmvr, s)) return rc;
  L.tiles = tiles; L.meta = meta;
  if (wp && numWp > 0) {
    if (int rc = g_hw.misc[2].reserve(numWp * sizeof(b200_wp))) return rc;
    B200_CUDA(cudaMemcpyAsync(g_hw.misc[2].p, wp, numWp * sizeof(b200_wp), cudaMemcpyHostToDevice, s));
    L.wp = g_hw.misc[2].as<b200_wp>();
  }
  if (int rc = fetch_list_meta(meta, L.cnt, MC_LISTS, "b200_mc_predict", s)) return rc;
  B200_CUDA(cudaMemsetAsync(g_hw.misc[7].p, 0, numDmvr * 8 + 64, s));
  memset(L.refs, 0, sizeof(L.refs)); for (size_t i = 0; i < ptrs.size(); i++) L.refs[i] = ptrs[i];
  for (int c = 0; c < 3; c++) L.refStride[c] = g->stride[c];
  L.pus = g_hw.misc[5].as<b200_pu>(); L.dmvrMv = dmvrMv ? g_hw.misc[7].as<int32_t>() : nullptr;
  StreamSet ss(s);
  if (int rc = launch_mc(L, ss)) return rc;
  if (int rc = download_planes(g, dst, L.dst, s)) return rc;
  if (dmvrMv && numDmvr) B200_CUDA(cudaMemcpyAsync(dmvrMv, g_hw.misc[7].p, numDmvr * 8, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
