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
  B200_CHECK(g->bitDepth >= 8 && g->bitDepth <= 12, "b200_k1_residual: bit depth %d unsupported", g->bitDepth);
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

// Samples a luma edge side of effective length n reads: n + 1 (its filters' reference sample), and p2/q2 for the decisions of lengths 1 and 2.
static int lf_reads(int n) { return n < 3 ? 3 : n + 1; }

// K3's flat pass (k3_deblock.cu) is exact only when no edge reads a sample that another edge of the same direction writes, and it reads no sample
// outside the plane.  One raster scan of a grid; returns false with the error set at the first edge that breaks a rule (include/vvdec_b200.h).
static bool lf_grid_legal(const b200_geom& g, const b200_lf_param* grid, int dir)
{
  const int W4 = g.width >> 2, H4 = g.height >> 2, extent = dir ? g.height : g.width;
  const char* name = dir ? "lfH" : "lfV";
  std::vector<int> prev(dir ? W4 : H4, -1), prevWQ(prev.size()), prevRQ(prev.size());   // per line: the last luma edge and its Q side's writes / reads
  for (int y4 = 0; y4 < H4; y4++)
    for (int x4 = 0; x4 < W4; x4++) {
      const b200_lf_param& e = grid[(size_t)y4 * W4 + x4];
      const int bs = e.bs & 0x3f, line = dir ? x4 : y4, pos = 4 * (dir ? y4 : x4);
      if (!bs) continue;
      if ((bs & 3) == 3 || ((bs >> 2) & 3) == 3 || (bs >> 4) == 3) { set_error("b200_lf_deblock: %s edge at (%d, %d): Bs 3", name, 4 * x4, 4 * y4); return false; }
      if (pos == 0) { set_error("b200_lf_deblock: %s edge at (%d, %d): Bs != 0 on the picture's border", name, 4 * x4, 4 * y4); return false; }
      if (!(bs & 3)) continue;                                  // chroma only: 4:2:0 chroma edges are 8 samples apart and read 4 per side
      int nP = (e.sideMaxFiltLength >> 4) & 7;
      const int nQ = e.sideMaxFiltLength & 7;
      const auto ok = [](int n) { return n == 1 || n == 2 || n == 3 || n == 5 || n == 7; };
      if (!ok(nP) || !ok(nQ)) { set_error("b200_lf_deblock: %s edge at (%d, %d): luma filter lengths %d/%d (1, 2, 3, 5 or 7)", name, 4 * x4, 4 * y4, nP, nQ); return false; }
      if (dir && (pos & (g.ctuSize - 1)) == 0 && nP > 3) nP = 3;   // a CTU row: the P side is never large
      const bool large = nP > 3 || nQ > 3;                       // the long filter runs a short side as length 3
      const int wP = large ? std::max(nP, 3) : nP, wQ = large ? std::max(nQ, 3) : nQ, rP = lf_reads(wP), rQ = lf_reads(wQ);
      if (pos < rP || pos + rQ > extent) { set_error("b200_lf_deblock: %s edge at (%d, %d): lengths %d/%d read outside the picture", name, 4 * x4, 4 * y4, nP, nQ); return false; }
      if (prev[line] >= 0 && (pos - prev[line] < prevWQ[line] + rP || pos - prev[line] < prevRQ[line] + wP)) {
        set_error("b200_lf_deblock: %s edge at (%d, %d): reads or writes samples the edge %d samples before it writes or reads", name, 4 * x4, 4 * y4, pos - prev[line]);
        return false;
      }
      prev[line] = pos; prevWQ[line] = wQ; prevRQ[line] = rQ;
    }
  return true;
}

B200_API int b200_lf_deblock(const b200_geom* g, int16_t* const planes[3], const b200_lf_param* lfV, const b200_lf_param* lfH,
                             const uint8_t* ctuSlice, const b200_lf_slice* slices, int numSlices, const b200_lf_seq* seq, int dirs)
{
  B200_CHECK(g && planes && lfV && lfH && slices, "b200_lf_deblock: null argument");
  B200_CHECK(numSlices >= 1 && numSlices <= 64, "b200_lf_deblock: numSlices %d out of range 1..64", numSlices);
  B200_CHECK(g->ctuSize == 32 || g->ctuSize == 64 || g->ctuSize == 128, "b200_lf_deblock: CTU size %d", g->ctuSize);
  // K3 filters 4:0:0 and 4:2:0 only; any other format would upload three planes and leave chroma unfiltered
  B200_CHECK(g->chromaFormat == 0 || g->chromaFormat == 1, "b200_lf_deblock: chromaFormat %d (only 0 = 4:0:0 and 1 = 4:2:0)", g->chromaFormat);
  B200_CHECK(g->bitDepth >= 8 && g->bitDepth <= 12, "b200_lf_deblock: bit depth %d (8..12)", g->bitDepth);
  B200_CHECK(g->width > 0 && g->height > 0 && !(g->width & 7) && !(g->height & 7), "b200_lf_deblock: picture %dx%d is not a multiple of 8", g->width, g->height);
  B200_CHECK(g->stride[0] >= g->width && (!g->chromaFormat || (g->stride[1] >= g->width / 2 && g->stride[2] >= g->width / 2)),
             "b200_lf_deblock: a plane stride is smaller than the plane's width");
  B200_CHECK(!(dirs & ~3), "b200_lf_deblock: dirs %d (bit 0 vertical, bit 1 horizontal edges)", dirs);
  B200_CHECK(!seq || !seq->ladfEnabled || (seq->ladfNumIntervals >= 2 && seq->ladfNumIntervals <= 5), "b200_lf_deblock: %d LADF intervals (2..5)", seq ? seq->ladfNumIntervals : 0);
  const size_t n4 = (size_t)((g->width + 3) >> 2) * ((g->height + 3) >> 2);
  const size_t nCtu = (size_t)((g->width + g->ctuSize - 1) / g->ctuSize) * ((g->height + g->ctuSize - 1) / g->ctuSize);
  for (size_t i = 0; ctuSlice && i < nCtu; i++) B200_CHECK(ctuSlice[i] < numSlices, "b200_lf_deblock: CTU %zu is in slice %d of %d", i, ctuSlice[i], numSlices);
  if (!lf_grid_legal(*g, lfV, 0) || !lf_grid_legal(*g, lfH, 1)) return B200_ERR_PARAM;
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

// The geometry K4 and K5 filter (include/vvdec_b200.h): 4:0:0 or 4:2:0, CTU 32 / 64 / 128, a picture of whole 8x8 units, and every plane's stride at
// least its width and a multiple of 4 (both kernels move 4 samples per 8-byte access, Cr included).  Returns false with the error set.
static bool k45_geom_ok(const char* fn, const b200_geom& g, int maxBitDepth)
{
  if (g.chromaFormat != 0 && g.chromaFormat != 1) { set_error("%s: chromaFormat %d (only 0 = 4:0:0 and 1 = 4:2:0)", fn, g.chromaFormat); return false; }
  if (g.ctuSize != 32 && g.ctuSize != 64 && g.ctuSize != 128) { set_error("%s: CTU size %d (32, 64 or 128)", fn, g.ctuSize); return false; }
  if (g.bitDepth < 8 || g.bitDepth > maxBitDepth) { set_error("%s: bit depth %d (8..%d)", fn, g.bitDepth, maxBitDepth); return false; }
  if (g.width <= 0 || g.height <= 0 || (g.width & 7) || (g.height & 7)) { set_error("%s: picture %dx%d is not a multiple of 8", fn, g.width, g.height); return false; }
  for (int c = 0; c < (g.chromaFormat ? 3 : 1); c++) {
    const int pw = c ? g.width >> 1 : g.width;
    if (g.stride[c] < pw || (g.stride[c] & 3)) { set_error("%s: plane %d stride %d (at least the plane width %d, a multiple of 4)", fn, c, g.stride[c], pw); return false; }
  }
  return true;
}

// SAO records and virtual boundaries: types 0..4 or OFF, BO bands 0..31, at most 3 boundaries per direction on the 8x8 grid strictly inside the picture.
static bool sao_records_ok(const b200_geom& g, const b200_sao_ctu* ctus, const b200_vb* vb)
{
  const size_t nCtu = (size_t)((g.width + g.ctuSize - 1) / g.ctuSize) * ((g.height + g.ctuSize - 1) / g.ctuSize);
  for (size_t i = 0; i < nCtu; i++)
    for (int c = 0; c < (g.chromaFormat ? 3 : 1); c++) {
      const int t = ctus[i].type[c];
      if (t != B200_SAO_OFF && t > B200_SAO_BO) { set_error("b200_sao_picture: CTU %zu component %d: type %d", i, c, t); return false; }
      if (t == B200_SAO_BO && ctus[i].band[c] > 31) { set_error("b200_sao_picture: CTU %zu component %d: band %d", i, c, ctus[i].band[c]); return false; }
    }
  if (!vb) return true;
  if (vb->numVer < 0 || vb->numVer > 3 || vb->numHor < 0 || vb->numHor > 3) { set_error("b200_sao_picture: %d / %d virtual boundaries (0..3 each)", vb->numVer, vb->numHor); return false; }
  for (int k = 0; k < vb->numVer; k++)
    if (vb->posX[k] <= 0 || vb->posX[k] >= g.width || (vb->posX[k] & 7)) { set_error("b200_sao_picture: vertical virtual boundary at x = %d", vb->posX[k]); return false; }
  for (int k = 0; k < vb->numHor; k++)
    if (vb->posY[k] <= 0 || vb->posY[k] >= g.height || (vb->posY[k] & 7)) { set_error("b200_sao_picture: horizontal virtual boundary at y = %d", vb->posY[k]); return false; }
  return true;
}

// ALF tables and records: every index inside its table, no undefined enable bit, and the padding forms the reference can produce (a corner is padded only
// where both adjacent sides are readable and the diagonal CTU exists; the wide chroma form only without CC-ALF on that component).
static bool alf_records_ok(const b200_geom& g, const b200_alf_ctu* ctus, const b200_alf_tables& T)
{
  const char* fn = "b200_alf_picture";
  if (T.numLumaSets < 16 || T.numLumaSets > 24) { set_error("%s: numLumaSets %d (16..24)", fn, T.numLumaSets); return false; }
  // the tables of a picture with several slices hold every slice's APS filters, so only the lower bounds are fixed
  if (T.numChromaAlts < 0) { set_error("%s: numChromaAlts %d", fn, T.numChromaAlts); return false; }
  for (int c = 0; c < 2; c++) if (T.numCc[c] < 0) { set_error("%s: numCc[%d] %d", fn, c, T.numCc[c]); return false; }
  const int ctusW = (g.width + g.ctuSize - 1) / g.ctuSize, ctusH = (g.height + g.ctuSize - 1) / g.ctuSize;
  for (int i = 0; i < ctusW * ctusH; i++) {
    const b200_alf_ctu& a = ctus[i];
    const int cx = i % ctusW, cy = i / ctusW, f = a.enable[0];
    if ((f & ~0x7f) || (a.enable[1] & ~3) || (a.enable[2] & ~3)) { set_error("%s: CTU %d: undefined enable bits %02x %02x %02x", fn, i, a.enable[0], a.enable[1], a.enable[2]); return false; }
    if ((f & 1) && a.lumaSet >= T.numLumaSets) { set_error("%s: CTU %d: lumaSet %d of %d", fn, i, a.lumaSet, T.numLumaSets); return false; }
    for (int c = 0; c < 2; c++) {
      if ((a.enable[1 + c] & 1) && a.chromaAlt[c] >= T.numChromaAlts) { set_error("%s: CTU %d: chromaAlt[%d] %d of %d", fn, i, c, a.chromaAlt[c], T.numChromaAlts); return false; }
      if (a.ccIdx[c] > T.numCc[c]) { set_error("%s: CTU %d: ccIdx[%d] %d of %d", fn, i, c, a.ccIdx[c], T.numCc[c]); return false; }
      if ((a.enable[1 + c] & B200_ALF_PAD_WIDE) && a.ccIdx[c]) { set_error("%s: CTU %d: PAD_WIDE with CC-ALF on component %d", fn, i, c + 1); return false; }
    }
    if ((f & B200_ALF_PAD_TL) && ((f & (B200_ALF_CLIP_TOP | B200_ALF_CLIP_LEFT)) || !cx || !cy)) { set_error("%s: CTU %d: PAD_TL with a clipped top / left side or on the picture's first CTU row / column", fn, i); return false; }
    if ((f & B200_ALF_PAD_BR) && ((f & (B200_ALF_CLIP_BOTTOM | B200_ALF_CLIP_RIGHT)) || cx == ctusW - 1 || cy == ctusH - 1)) { set_error("%s: CTU %d: PAD_BR with a clipped bottom / right side or on the picture's last CTU row / column", fn, i); return false; }
  }
  return true;
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
  if (!k45_geom_ok("b200_sao_picture", *g, 12) || !sao_records_ok(*g, ctus, vb)) return B200_ERR_PARAM;
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  SaoLaunch L; L.geom = *g;
  if (vb) L.vb = *vb; else memset(&L.vb, 0, sizeof(L.vb));
  if (int rc = upload_src_alloc_dst(g, src, L.src, L.dst, s)) return rc;
  const size_t nCtu = (size_t)((g->width + g->ctuSize - 1) / g->ctuSize) * ((g->height + g->ctuSize - 1) / g->ctuSize);
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
  B200_CHECK(g->bitDepth >= 8 && g->bitDepth <= 12, "b200_intra_reconstruct: bit depth %d unsupported", g->bitDepth);
  const int nPl = g->chromaFormat ? 3 : 1;
  for (size_t i = 0; i < numTus; i++) {                      // kernel-level wrapper: records are checked here (the picture path checks on the device)
    const b200_intra_tu& t = tus[i];
    const int w = 1 << t.log2w, h = 1 << t.log2h, pw = t.comp ? g->width >> 1 : g->width, ph = t.comp ? g->height >> 1 : g->height, unit = t.comp ? 2 : 4;
    const bool inCtu = intra_record_in_ctu(t, intra_ctu_log2(*g));
    if (t.flags & B200_INTRA_ISP) {
      B200_CHECK(intra_isp_record_ok(t, i ? &tus[i - 1] : nullptr, g->width, g->height), "b200_intra_reconstruct: record %zu: bad ISP region", i);
      B200_CHECK(inCtu, "b200_intra_reconstruct: intra block record %zu is not inside one CTU", i);
      continue;
    }
    B200_CHECK(t.comp < nPl && t.log2w >= 2 && t.log2w <= 6 && t.log2h >= 1 && t.log2h <= 6 && t.x + w <= pw && t.y + h <= ph && !(t.x % unit) && !(t.y % unit),
               "b200_intra_reconstruct: record %zu: bad geometry", i);
    B200_CHECK(inCtu, "b200_intra_reconstruct: intra block record %zu is not inside one CTU", i);
    B200_CHECK(t.mode <= B200_INTRA_MDLM_T && t.multiRefIdx <= 2 && (!t.multiRefIdx || !t.comp), "b200_intra_reconstruct: record %zu: bad mode / reference line", i);
    B200_CHECK(!t.ciip || (t.ciip <= 3 && t.mode == B200_INTRA_PLANAR), "b200_intra_reconstruct: record %zu: bad CIIP block", i);
    B200_CHECK(t.mode < B200_INTRA_LM || (t.comp && t.log2w <= 5 && t.log2h <= 5 && t.lmAbove <= w && t.lmLeft <= h && (!(t.flags & B200_INTRA_LM_ABOVE) || t.y >= 2) && (!(t.flags & B200_INTRA_LM_LEFT) || t.x >= 2)
                                        && t.x + std::max(w, 2 * (int)t.lmAbove) <= pw && t.y + std::max(h, 2 * (int)t.lmLeft) <= ph), "b200_intra_reconstruct: record %zu: bad CCLM block", i);
    B200_CHECK(t.mode != B200_INTRA_MIP || (!t.comp && !t.multiRefIdx && (t.mip & 0x7f) < ((w == 4 && h == 4) ? 16 : (w == 4 || h == 4 || (w == 8 && h == 8)) ? 8 : 6)),
               "b200_intra_reconstruct: record %zu: bad MIP mode", i);
    B200_CHECK(t.numAbove <= 2 * w / unit && t.numLeft <= 2 * h / unit && (!t.numAbove || t.y > t.multiRefIdx) && (!t.numLeft || t.x > t.multiRefIdx)
               && (!(t.flags & B200_INTRA_AVAIL_TL) || (t.x > t.multiRefIdx && t.y > t.multiRefIdx)) && t.x + (int)t.numAbove * unit <= pw && t.y + (int)t.numLeft * unit <= ph,
               "b200_intra_reconstruct: record %zu: availability outside the picture", i);
  }
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
  if (!k45_geom_ok("b200_alf_picture", *g, 10) || !alf_records_ok(*g, ctus, *T)) return B200_ERR_PARAM;
  if (int rc = ensure_device()) return rc;
  if (int rc = g_hw.init()) return rc;
  cudaStream_t s = g_hw.stream;
  AlfLaunch L; L.geom = *g;
  if (int rc = upload_src_alloc_dst(g, src, L.src, L.dst, s)) return rc;
  const size_t nCtu = (size_t)((g->width + g->ctuSize - 1) / g->ctuSize) * ((g->height + g->ctuSize - 1) / g->ctuSize);
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
  // K2 predicts 4:0:0 and 4:2:0 only; any other format would upload three planes and leave chroma unwritten
  B200_CHECK(g->chromaFormat == 0 || g->chromaFormat == 1, "b200_mc_predict: chromaFormat %d (only 0 = 4:0:0 and 1 = 4:2:0)", g->chromaFormat);
  B200_CHECK(g->bitDepth >= 8 && g->bitDepth <= 12, "b200_mc_predict: bit depth %d (8..12)", g->bitDepth);
  B200_CHECK(g->width > 0 && g->height > 0 && g->stride[0] >= g->width && (!g->chromaFormat || (g->stride[1] >= g->width / 2 && g->stride[2] >= g->width / 2)),
             "b200_mc_predict: a plane stride is smaller than the plane's width");
  B200_CHECK(numSlots >= 1 && numSlots <= B200_MAX_SLOTS, "b200_mc_predict: numSlots %d", numSlots);
  B200_CHECK(numPus < (1u << 26), "b200_mc_predict: too many PUs");
  for (size_t i = 0; i < numPus; i++) {
    B200_CHECK(pus[i].refSlot[0] < numSlots && pus[i].refSlot[1] < numSlots && (pus[i].refSlot[0] >= 0 || pus[i].refSlot[1] >= 0), "b200_mc_predict: PU %zu has invalid reference slots", i);
    B200_CHECK(!((pus[i].flags & B200_PU_DMVR) && g->bitDepth > 10), "b200_mc_predict: DMVR needs bit depth <= 10 (as the reference)");
  }
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
    B200_CHECK(numWp <= 255, "b200_mc_predict_wp: at most 255 weighted-prediction entries");
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
