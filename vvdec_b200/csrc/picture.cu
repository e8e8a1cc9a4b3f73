// picture.cu — picture-level context: device-resident DPB, work-list arenas, and the per-picture kernel chain
// (the device replacement of DecLibRecon::decompressPicture's CTU task graph, reference DecoderLib/DecLibRecon.cpp:429-682).
#include "common.cuh"
#include <string.h>
#include <vector>

namespace b200 {

static inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

struct Arena {
  DevBuf buf;                       // one allocation, sub-allocated per picture
  // device views
  const b200_pu* pus = nullptr; size_t numPus = 0; const uint32_t* tiles = nullptr; int* mcMeta = nullptr;   // device lists built by bucket.cu
  int* hMeta = nullptr;             // pinned host copy of both meta blocks (list lengths + error bits), valid once `uploaded` has fired
  const b200_tu* tus = nullptr; size_t numTus = 0; const uint32_t* tuIdx = nullptr; int* tuMeta = nullptr; const int16_t* coefs = nullptr; const int32_t* scaling = nullptr;
  const b200_lf_param *lfV = nullptr, *lfH = nullptr; const uint8_t* ctuSlice = nullptr; LfSliceTab lfSlices; b200_lf_seq lfSeq;
  const b200_sao_ctu* sao = nullptr; b200_vb vb;
  const b200_alf_ctu* alf = nullptr; const int16_t *lumaCoeff = nullptr, *lumaClip = nullptr, *chromaCoeff = nullptr, *chromaClip = nullptr, *cc[2] = {nullptr, nullptr};
  int32_t* dmvrMv = nullptr; size_t numDmvr = 0;
  const b200_wp* wp = nullptr;
  const b200_lmcs* lmcs = nullptr; const int16_t* lmcsInv = nullptr; const b200_lmcs_vpdu* lmcsVpdus = nullptr; int* lmcsScale = nullptr; bool lmcsChromaAdj = false;
  int16_t* given[3] = {nullptr, nullptr, nullptr};
  const b200_intra_tu* intraTus = nullptr; size_t numIntraTus = 0; int* intraOwner[3] = {nullptr, nullptr, nullptr}; int intraOwnerStride[3] = {0, 0, 0}; size_t intraOwnerBytes[3] = {0, 0, 0}; int* intraSync = nullptr; int* intraOrder = nullptr;   // K6
  int dstSlot = 0, flags = 0;
  bool ciipResi = false;             // a CIIP block takes a residual: its residual-plane area is cleared before K1 (k6_intra.cu)
  bool valid = false;
  cudaEvent_t uploaded = nullptr, done = nullptr; bool donePending = false;   // H2D finished / kernels reading this arena finished
};

}  // namespace b200

using namespace b200;

struct CtxProf : b200::KProf {
  struct Rec { int family; cudaEvent_t a, b; };
  std::vector<Rec> recs; std::vector<cudaEvent_t> pool; Rec cur{};
  cudaEvent_t get() { cudaEvent_t e; if (!pool.empty()) { e = pool.back(); pool.pop_back(); } else cudaEventCreate(&e); return e; }
  void begin(int f, cudaStream_t s) override { cur.family = f; cur.a = get(); cur.b = get(); cudaEventRecord(cur.a, s); }
  void end(int, cudaStream_t s) override { cudaEventRecord(cur.b, s); recs.push_back(cur); }
};

struct b200_ctx {
  b200_geom g;
  CtxProf prof; bool profiling = false;
  int numSlots = 0, numArenas = 0, device = 0;
  cudaStream_t stream = nullptr, copyStream = nullptr, upStream = nullptr;   // kernels / frame output D2H / work-list H2D
  StreamSet ss;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  std::vector<cudaEvent_t> readDone; std::vector<char> readPending;   // per picture buffer: an async output (maybe) still reads it (mark_read)
  std::vector<cudaStream_t> readStream;                              // the stream readDone was last recorded on
  cudaEvent_t ticketEv[16]; cudaEvent_t finalEv = nullptr; int nextTicket = 0;
  DevBuf outStage[2]; int nextStage = 0;   // converted output frames (pyuv / 8 bit) waiting for their D2H copy
  size_t planeBytes[3] = {0, 0, 0}, picBytes = 0;
  std::vector<int16_t*> bufs;          // numSlots + 2 picture buffers
  std::vector<int> slotBuf;            // slot -> buffer index
  int work[2] = {0, 0};                // indices of the two work buffers
  std::vector<Arena> arenas;
  int nextArena = 0;
  long long launches = 0;
  DevBuf grainStage[2], grainTab;    // b200_get_frame_grain_async: grained copy of the frame, device copies of the tables + block seeds
  struct HostStage { void* p = nullptr; size_t cap = 0; cudaEvent_t copied = nullptr; bool pending = false; } grainHost[2];   // pinned copies of the caller's tables
  DevBuf resiBuf;                    // residual planes of intra CUs (K1 -> K6), allocated with the first picture that carries intra blocks
  DevBuf hashBuf;                    // b200_frame_hash_async: accumulators + digest per ticket

  DevPlanes planes(int buf) const {
    DevPlanes d; char* b = reinterpret_cast<char*>(bufs[buf]);
    d.p[0] = reinterpret_cast<int16_t*>(b); d.p[1] = reinterpret_cast<int16_t*>(b + planeBytes[0]); d.p[2] = reinterpret_cast<int16_t*>(b + planeBytes[0] + planeBytes[1]);
    for (int c = 0; c < 3; c++) d.stride[c] = g.stride[c];
    return d;
  }
};

extern "C" {

static int copy2d_host(void* dst, size_t dpitch, const void* src, size_t spitch, size_t wBytes, size_t h, cudaMemcpyKind kind, cudaStream_t s);
// a contiguous copy between caller memory and the device (see copy2d_host: the caller's array may start in a page registered for another array)
static inline int copy_host(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t s) { return copy2d_host(dst, bytes, src, bytes, bytes, 1, kind, s); }

// Ordering of the picture buffers and their asynchronous readers (the output calls): readDone[buf] is where the last reader of buffer `buf` is done.  A
// reader on stream s records it after its own work; when a reader on another stream is still pending, s first waits for that one, so the one event covers
// both (s's later work then waits for it too).  b200_pic_run (for its two work buffers) and b200_ctx_load_slot* wait for readDone before they write a buffer.
static int mark_read(b200_ctx* c, int buf, cudaStream_t s)
{
  if (c->readPending[buf] && c->readStream[buf] != s) B200_CUDA(cudaStreamWaitEvent(s, c->readDone[buf], 0));
  B200_CUDA(cudaEventRecord(c->readDone[buf], s));
  c->readPending[buf] = 1; c->readStream[buf] = s;
  return 0;
}

static int wait_readers(b200_ctx* c, int buf)
{
  if (c->readPending[buf]) { B200_CUDA(cudaStreamWaitEvent(c->stream, c->readDone[buf], 0)); c->readPending[buf] = 0; }
  return 0;
}

B200_API int b200_ctx_create(b200_ctx** out, const b200_geom* g, int numSlots, int numArenas, int device)
{
  B200_CHECK(out && g, "b200_ctx_create: null argument");
  B200_CHECK(numSlots >= 1 && numSlots <= B200_MAX_SLOTS && numArenas >= 1 && numArenas <= 256, "b200_ctx_create: numSlots %d / numArenas %d out of range", numSlots, numArenas);
  if (const char* why = geom_problem(*g, 12, 1)) { set_error("b200_ctx_create: %s", why); return B200_ERR_PARAM; }
  if (int rc = ensure_device()) return rc;
  if (device >= 0) B200_CUDA(cudaSetDevice(device));
  b200_ctx* c = new b200_ctx;
  c->g = *g; c->numSlots = numSlots; c->numArenas = numArenas;
  B200_CUDA(cudaGetDevice(&c->device));
  B200_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  B200_CUDA(cudaStreamCreateWithFlags(&c->copyStream, cudaStreamNonBlocking));
  B200_CUDA(cudaStreamCreateWithFlags(&c->upStream, cudaStreamNonBlocking));
  c->ss.main = c->stream; c->ss.nAux = 3;
  B200_CUDA(cudaEventCreateWithFlags(&c->ss.forkEv, cudaEventDisableTiming));
  for (int k = 0; k < c->ss.nAux; k++) { B200_CUDA(cudaStreamCreateWithFlags(&c->ss.aux[k], cudaStreamNonBlocking)); B200_CUDA(cudaEventCreateWithFlags(&c->ss.joinEv[k], cudaEventDisableTiming)); }
  B200_CUDA(cudaEventCreate(&c->ev[0])); B200_CUDA(cudaEventCreate(&c->ev[1]));
  B200_CUDA(cudaEventCreateWithFlags(&c->finalEv, cudaEventDisableTiming));
  for (auto& e : c->ticketEv) B200_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (int k = 0; k < 3; k++) c->planeBytes[k] = (k == 0 || g->chromaFormat) ? align256((size_t)g->stride[k] * (k ? g->height >> 1 : g->height) * 2) : 0;
  c->picBytes = c->planeBytes[0] + c->planeBytes[1] + c->planeBytes[2];
  c->bufs.resize(numSlots + 2); c->slotBuf.resize(numSlots);
  c->readDone.resize(numSlots + 2); c->readPending.assign(numSlots + 2, 0); c->readStream.assign(numSlots + 2, nullptr);
  for (auto& e : c->readDone) B200_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto& h : c->grainHost) B200_CUDA(cudaEventCreateWithFlags(&h.copied, cudaEventDisableTiming));
  for (int i = 0; i < numSlots + 2; i++) { B200_CUDA(cudaMalloc(&c->bufs[i], c->picBytes)); B200_CUDA(cudaMemset(c->bufs[i], 0, c->picBytes)); }
  for (int s = 0; s < numSlots; s++) c->slotBuf[s] = s;
  c->work[0] = numSlots; c->work[1] = numSlots + 1;
  c->arenas.resize(numArenas);
  for (auto& A : c->arenas) { B200_CUDA(cudaEventCreateWithFlags(&A.uploaded, cudaEventDisableTiming)); B200_CUDA(cudaEventCreateWithFlags(&A.done, cudaEventDisableTiming)); B200_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&A.hMeta), (2 * LM_INTS + 4) * sizeof(int), cudaHostAllocDefault)); }
  *out = c;
  return 0;
}

B200_API void b200_ctx_destroy(b200_ctx* c)
{
  if (!c) return;
  cudaStreamSynchronize(c->stream); cudaStreamSynchronize(c->copyStream); cudaStreamSynchronize(c->upStream);
  for (auto& A : c->arenas) { cudaEventDestroy(A.uploaded); cudaEventDestroy(A.done); if (A.hMeta) cudaFreeHost(A.hMeta); }
  cudaStreamDestroy(c->upStream);
  for (auto p : c->bufs) cudaFree(p);
  for (auto e : c->readDone) cudaEventDestroy(e);
  for (auto e : c->ticketEv) cudaEventDestroy(e);
  for (auto& h : c->grainHost) { cudaEventDestroy(h.copied); if (h.p) cudaFreeHost(h.p); }
  cudaEventDestroy(c->finalEv); cudaStreamDestroy(c->copyStream);
  for (int k = 0; k < c->ss.nAux; k++) { cudaStreamSynchronize(c->ss.aux[k]); cudaStreamDestroy(c->ss.aux[k]); cudaEventDestroy(c->ss.joinEv[k]); }
  cudaEventDestroy(c->ss.forkEv);
  cudaEventDestroy(c->ev[0]); cudaEventDestroy(c->ev[1]);
  cudaStreamDestroy(c->stream);
  delete c;
}

B200_API int b200_ctx_load_slot(b200_ctx* c, int slot, const int16_t* const planes[3])
{
  B200_CHECK(c && planes && slot >= 0 && slot < c->numSlots, "b200_ctx_load_slot: bad argument");
  if (int rc = wait_readers(c, c->slotBuf[slot])) return rc;
  DevPlanes d = c->planes(c->slotBuf[slot]);
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++)
    if (int rc = copy_host(d.p[k], planes[k], (size_t)c->g.stride[k] * (k ? c->g.height >> 1 : c->g.height) * 2, cudaMemcpyHostToDevice, c->stream)) return rc;
  B200_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

B200_API int b200_pic_upload(b200_ctx* c, const b200_picture* p)
{
  B200_CHECK(c && p, "b200_pic_upload: null argument");
  B200_CHECK(p->dstSlot >= 0 && p->dstSlot < c->numSlots, "b200_pic_upload: dstSlot %d", p->dstSlot);
  B200_CHECK(!(p->flags & B200_PIC_DEBLOCK) || (p->lfV && p->lfH && p->lfSlices && p->numLfSlices >= 1 && p->numLfSlices <= 64), "b200_pic_upload: deblocking data missing");
  B200_CHECK(!(p->flags & B200_PIC_SAO) || p->sao, "b200_pic_upload: SAO data missing");
  B200_CHECK(!(p->flags & B200_PIC_ALF) || (p->alf && p->alfTabs), "b200_pic_upload: ALF data missing");
  // the O(1) rules of b200_sao_picture / b200_alf_picture (rules.cuh); the CTU records are checked on the device
  const char* why = nullptr;
  if (p->flags & (B200_PIC_SAO | B200_PIC_ALF)) why = geom_problem(c->g, (p->flags & B200_PIC_ALF) ? 10 : 12, 4);
  if (!why && (p->flags & B200_PIC_ALF)) why = alf_tables_problem(*p->alfTabs, 255);   // a picture's tables hold every slice's APS sets
  if (!why && (p->flags & B200_PIC_SAO) && p->vb) why = vb_problem(*p->vb, c->g.width, c->g.height);
  if (why) { set_error("b200_pic_upload: %s", why); return B200_ERR_PARAM; }
  B200_CHECK(p->numPus < (1u << 26) && p->numTus < (1u << 31), "b200_pic_upload: too many records");
  B200_CHECK(p->numWp >= 0 && p->numWp <= 255 && (p->wp || !p->numWp), "b200_pic_upload: weighted-prediction table (at most 255 entries)");
  B200_CHECK(!(p->flags & B200_PIC_LMCS) || (p->lmcs && p->lmcs->invLUT && (!p->lmcs->chromaAdj || p->lmcs->vpdus)), "b200_pic_upload: LMCS data missing");
  if (p->flags & B200_PIC_LMCS) if (const char* why = lmcs_model_problem(*p->lmcs, c->g.bitDepth)) { set_error("b200_pic_upload: %s", why); return B200_ERR_PARAM; }
  B200_CHECK(!p->numIntraTus || (p->intraTus && p->numIntraTus < (1u << 30)), "b200_pic_upload: intra list missing");
  B200_CUDA(cudaSetDevice(c->device));
  const int ai = c->nextArena; c->nextArena = (c->nextArena + 1) % c->numArenas;
  Arena& A = c->arenas[ai];
  A.valid = false;                                                    // until every copy of this upload has been enqueued
  const b200_geom& g = c->g;
  const size_t n4 = (size_t)((g.width + 3) >> 2) * ((g.height + 3) >> 2);
  const size_t nCtu = (size_t)((g.width + g.ctuSize - 1) / g.ctuSize) * ((g.height + g.ctuSize - 1) / g.ctuSize);
  // No per-record work on the host: the caller's arrays are copied as they are; the records are validated and sorted into the
  // kernels' work lists on the device (bucket.cu), errors surface in b200_pic_run.
  const size_t capTiles = mc_tile_capacity(g, 0);
  const b200_alf_tables* T = p->alfTabs;
  const size_t nL = (p->flags & B200_PIC_ALF) ? (size_t)T->numLumaSets * 1300 : 0, nC = (p->flags & B200_PIC_ALF) ? (size_t)T->numChromaAlts * 7 : 0;
  const size_t n0 = (p->flags & B200_PIC_ALF) ? (size_t)T->numCc[0] * 7 : 0, n1 = (p->flags & B200_PIC_ALF) ? (size_t)T->numCc[1] * 7 : 0;
  // ---- layout ----
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += align256(bytes + 16); return o; };
  const size_t oPus = take(p->numPus * sizeof(b200_pu)), oT = take(capTiles * 4), oMeta = take(2 * LM_INTS * sizeof(int)), oIdx = take(p->numTus * 4);
  const size_t oTus = take(p->numTus * sizeof(b200_tu)), oCoef = take(p->numCoefs * 2), oScal = take(p->numScaling * 4);
  const size_t oLfV = take((p->flags & B200_PIC_DEBLOCK) ? n4 * 6 : 0), oLfH = take((p->flags & B200_PIC_DEBLOCK) ? n4 * 6 : 0), oCs = take(nCtu);
  const size_t oSao = take((p->flags & B200_PIC_SAO) ? nCtu * sizeof(b200_sao_ctu) : 0);
  const size_t oAlf = take((p->flags & B200_PIC_ALF) ? nCtu * sizeof(b200_alf_ctu) : 0), oTab = take((2 * nL + 2 * nC + n0 + n1) * 2);
  const size_t oDm = take(p->numDmvr * 8);
  const size_t oWp = take((size_t)p->numWp * sizeof(b200_wp));
  const bool lm = p->flags & B200_PIC_LMCS;
  const int vs = g.ctuSize == 128 ? 64 : g.ctuSize; const size_t nVpdu = (size_t)((g.width + vs - 1) / vs) * ((g.height + vs - 1) / vs);
  const size_t oLm = take(lm ? sizeof(b200_lmcs) : 0), oLmLut = take(lm ? sizeof(int16_t) << g.bitDepth : 0), oLmVp = take(lm ? nVpdu * sizeof(b200_lmcs_vpdu) : 0), oLmSc = take(lm ? nVpdu * sizeof(int) : 0);
  const bool hasGiven = p->given[0] != nullptr;
  const size_t oGiven = take(hasGiven ? c->picBytes : 0);
  size_t oOwn[3] = {0, 0, 0}, ownBytes[3] = {0, 0, 0}; int ownStride[3] = {0, 0, 0};
  const size_t oIntra = take(p->numIntraTus * sizeof(b200_intra_tu)), oSync = take(p->numIntraTus ? (p->numIntraTus + 2) * sizeof(int) : 0), oOrder = take(p->numIntraTus ? intra_order_ints(g, p->numIntraTus) * sizeof(int) : 0);
  for (int k = 0; k < (g.chromaFormat ? 3 : 1) && p->numIntraTus; k++) {
    const int pw = k ? g.width >> 1 : g.width, ph = k ? g.height >> 1 : g.height, unit = k ? 2 : 4;
    ownStride[k] = (pw + unit - 1) / unit; ownBytes[k] = (size_t)ownStride[k] * ((ph + unit - 1) / unit) * sizeof(int); oOwn[k] = take(ownBytes[k]);
  }
  if (p->numIntraTus) if (int rc = c->resiBuf.reserve(c->picBytes)) return rc;
  if (off > A.buf.cap) { B200_CUDA(cudaStreamSynchronize(c->stream)); B200_CUDA(cudaStreamSynchronize(c->upStream)); A.donePending = false; }   // realloc: nothing may still use the old buffer
  if (int rc = A.buf.reserve(off)) return rc;
  char* base = A.buf.as<char>();
  cudaStream_t s = c->upStream;                                       // H2D on its own stream: overlaps the kernels of earlier pictures
  if (A.donePending) { B200_CUDA(cudaStreamWaitEvent(s, A.done, 0)); A.donePending = false; }   // kernels of the arena's previous picture
  auto h2d = [&](size_t o, const void* src, size_t bytes) -> int { if (bytes) if (int rc = copy_host(base + o, src, bytes, cudaMemcpyHostToDevice, s)) return rc; return 0; };
  if (int rc = h2d(oPus, p->pus, p->numPus * sizeof(b200_pu))) return rc;
  if (int rc = h2d(oTus, p->tus, p->numTus * sizeof(b200_tu))) return rc;
  if (int rc = h2d(oCoef, p->coefs, p->numCoefs * 2)) return rc;
  if (int rc = h2d(oScal, p->scaling, p->numScaling * 4)) return rc;
  if (p->flags & B200_PIC_DEBLOCK) {
    if (int rc = h2d(oLfV, p->lfV, n4 * 6)) return rc;
    if (int rc = h2d(oLfH, p->lfH, n4 * 6)) return rc;
    if (p->ctuSlice) if (int rc = h2d(oCs, p->ctuSlice, nCtu)) return rc;
    memset(&A.lfSlices, 0, sizeof(A.lfSlices)); memcpy(A.lfSlices.s, p->lfSlices, p->numLfSlices * sizeof(b200_lf_slice));
    if (p->lfSeq) A.lfSeq = *p->lfSeq; else memset(&A.lfSeq, 0, sizeof(A.lfSeq));
  }
  if (p->flags & B200_PIC_SAO) { if (int rc = h2d(oSao, p->sao, nCtu * sizeof(b200_sao_ctu))) return rc; if (p->vb) A.vb = *p->vb; else memset(&A.vb, 0, sizeof(A.vb)); }
  if (p->flags & B200_PIC_ALF) {
    if (int rc = h2d(oAlf, p->alf, nCtu * sizeof(b200_alf_ctu))) return rc;
    size_t o = oTab;
    auto up = [&](const int16_t* src, size_t n, const int16_t*& view) -> int { view = reinterpret_cast<const int16_t*>(base + o); int rc = h2d(o, src, n * 2); o += n * 2; return rc; };
    if (int rc = up(T->lumaCoeff, nL, A.lumaCoeff)) return rc;
    if (int rc = up(T->lumaClip, nL, A.lumaClip)) return rc;
    if (int rc = up(T->chromaCoeff, nC, A.chromaCoeff)) return rc;
    if (int rc = up(T->chromaClip, nC, A.chromaClip)) return rc;
    if (int rc = up(T->ccCoeff[0], n0, A.cc[0])) return rc;
    if (int rc = up(T->ccCoeff[1], n1, A.cc[1])) return rc;
  }
  if (int rc = h2d(oWp, p->wp, (size_t)p->numWp * sizeof(b200_wp))) return rc;
  A.wp = p->numWp ? reinterpret_cast<const b200_wp*>(base + oWp) : nullptr;
  if (lm) {
    if (int rc = h2d(oLm, p->lmcs, sizeof(b200_lmcs))) return rc;
    if (int rc = h2d(oLmLut, p->lmcs->invLUT, sizeof(int16_t) << g.bitDepth)) return rc;
    if (p->lmcs->chromaAdj) if (int rc = h2d(oLmVp, p->lmcs->vpdus, nVpdu * sizeof(b200_lmcs_vpdu))) return rc;
    A.lmcs = reinterpret_cast<const b200_lmcs*>(base + oLm); A.lmcsInv = reinterpret_cast<const int16_t*>(base + oLmLut);
    A.lmcsVpdus = reinterpret_cast<const b200_lmcs_vpdu*>(base + oLmVp); A.lmcsScale = reinterpret_cast<int*>(base + oLmSc); A.lmcsChromaAdj = p->lmcs->chromaAdj != 0;
  } else { A.lmcs = nullptr; A.lmcsChromaAdj = false; }
  if (hasGiven) {
    size_t o = oGiven;
    for (int k = 0; k < (g.chromaFormat ? 3 : 1); k++) {
      A.given[k] = reinterpret_cast<int16_t*>(base + o);
      if (int rc = h2d(o, p->given[k], (size_t)g.stride[k] * (k ? g.height >> 1 : g.height) * 2)) return rc;
      o += c->planeBytes[k];
    }
  } else A.given[0] = A.given[1] = A.given[2] = nullptr;
  A.pus = reinterpret_cast<const b200_pu*>(base + oPus); A.numPus = p->numPus;
  A.tus = reinterpret_cast<const b200_tu*>(base + oTus); A.numTus = p->numTus;
  A.coefs = reinterpret_cast<const int16_t*>(base + oCoef); A.scaling = reinterpret_cast<const int32_t*>(base + oScal);
  A.lfV = reinterpret_cast<const b200_lf_param*>(base + oLfV); A.lfH = reinterpret_cast<const b200_lf_param*>(base + oLfH);
  A.ctuSlice = p->ctuSlice ? reinterpret_cast<const uint8_t*>(base + oCs) : nullptr;
  A.sao = reinterpret_cast<const b200_sao_ctu*>(base + oSao); A.alf = reinterpret_cast<const b200_alf_ctu*>(base + oAlf);
  A.dmvrMv = p->numDmvr ? reinterpret_cast<int32_t*>(base + oDm) : nullptr; A.numDmvr = p->numDmvr;
  if (p->numDmvr) B200_CUDA(cudaMemsetAsync(base + oDm, 0, p->numDmvr * 8, s));   // entries of non-DMVR CUs stay zero, like m_dmvrMvCache users expect
  if (int rc = h2d(oIntra, p->intraTus, p->numIntraTus * sizeof(b200_intra_tu))) return rc;
  A.intraTus = reinterpret_cast<const b200_intra_tu*>(base + oIntra); A.numIntraTus = p->numIntraTus; A.intraSync = reinterpret_cast<int*>(base + oSync); A.intraOrder = reinterpret_cast<int*>(base + oOrder);
  for (int k = 0; k < 3; k++) { A.intraOwner[k] = ownBytes[k] ? reinterpret_cast<int*>(base + oOwn[k]) : nullptr; A.intraOwnerStride[k] = ownStride[k]; A.intraOwnerBytes[k] = ownBytes[k]; }
  A.ciipResi = false;
  for (size_t i = 0; i < p->numIntraTus && !A.ciipResi; i++) { const b200_intra_tu& t = p->intraTus[i]; A.ciipResi = t.ciip && !(t.flags & B200_INTRA_ISP) && (t.flags & B200_INTRA_ADD_RESI); }
  A.dstSlot = p->dstSlot; A.flags = p->flags; A.valid = true;
  // work lists: validated and bucketed on the device, behind the copies
  A.mcMeta = reinterpret_cast<int*>(base + oMeta); A.tuMeta = A.mcMeta + LM_INTS;
  if (int rc = launch_mc_bucket(reinterpret_cast<const b200_pu*>(base + oPus), p->numPus, reinterpret_cast<uint32_t*>(base + oT), capTiles, A.mcMeta, g, c->numSlots, p->numWp, p->numDmvr, s)) return rc;
  if (int rc = launch_tu_bucket(reinterpret_cast<const b200_tu*>(base + oTus), p->numTus, reinterpret_cast<uint32_t*>(base + oIdx), A.tuMeta, g, p->numCoefs, p->numScaling, s)) return rc;
  A.tiles = reinterpret_cast<const uint32_t*>(base + oT); A.tuIdx = reinterpret_cast<const uint32_t*>(base + oIdx);
  c->launches += 4;
  {
    const bool alfOn = p->flags & B200_PIC_ALF, any = (p->flags & (B200_PIC_SAO | B200_PIC_ALF)) || ((p->flags & B200_PIC_DEBLOCK) && p->ctuSlice);
    if (int rc = launch_ctu_validate((p->flags & B200_PIC_SAO) ? A.sao : nullptr, alfOn ? A.alf : nullptr, (p->flags & B200_PIC_DEBLOCK) ? A.ctuSlice : nullptr, (int)nCtu,
                                     ctu_limits(g, alfOn ? T : nullptr, p->numLfSlices), A.mcMeta, s)) return rc;
    if (any) c->launches += 1;
  }
  if (A.numIntraTus) { if (int rc = launch_intra_validate(A.intraTus, A.numIntraTus, g, A.mcMeta, s)) return rc; c->launches += 1; }
  if (A.lmcsChromaAdj) { if (int rc = launch_lmcs_validate(A.lmcsVpdus, g, A.mcMeta, s)) return rc; c->launches += 1; }
  B200_CUDA(cudaMemcpyAsync(A.hMeta, A.mcMeta, 2 * LM_INTS * sizeof(int), cudaMemcpyDeviceToHost, s));   // list lengths for b200_pic_run's grids
  B200_CUDA(cudaEventRecord(A.uploaded, s));
  return ai;
}

B200_API int b200_pic_run(b200_ctx* c, int ai)
{
  B200_CHECK(c && ai >= 0 && ai < c->numArenas && c->arenas[ai].valid, "b200_pic_run: bad arena %d", ai);
  B200_CUDA(cudaSetDevice(c->device));
  Arena& A = c->arenas[ai];
  cudaStream_t s = c->stream;
  // the grids are sized from the list lengths the bucketing kernels produced: the host waits for this picture's upload (a caller that
  // uploads picture n+1 before it runs picture n never waits here)
  B200_CUDA(cudaEventSynchronize(A.uploaded));
  B200_CHECK(!(A.hMeta[LM_ERR] & 1), "b200_pic_run: the picture's PU list holds an invalid record (reference slots, block size or flag combination)");
  B200_CHECK(!(A.hMeta[LM_ERR] & 2), "b200_pic_run: more MC tiles than the picture can hold (overlapping PUs?)");
  B200_CHECK(!(A.hMeta[LM_ERR] & 8), "b200_pic_run: an intra block record is invalid (geometry, mode, or availability reaching outside the picture)");
  B200_CHECK(!(A.hMeta[LM_ERR] & 4), "b200_pic_run: a CTU record (SAO type / band, ALF filter index or clip / pad flags, slice index) is out of range");
  B200_CHECK(!(A.hMeta[LM_ERR] & 16), "b200_pic_run: an LMCS VPDU record is invalid (CU origin outside the picture or not at or above-left of its VPDU in the same CTU, or an available neighbour outside the picture)");
  B200_CHECK(!A.hMeta[LM_INTS + LM_ERR], "b200_pic_run: the picture's TU list holds an invalid record");
  B200_CUDA(cudaStreamWaitEvent(s, A.uploaded, 0));
  const b200_geom& g = c->g;
  int cur = c->work[0], other = c->work[1];
  for (int b : {cur, other}) if (int rc = wait_readers(c, b)) return rc;   // async outputs still reading these buffers
  DevPlanes P = c->planes(cur);
  // 0. pre-reconstructed (intra stand-in) samples
  if (A.given[0]) {
    for (int k = 0; k < (g.chromaFormat ? 3 : 1); k++)
      B200_CUDA(cudaMemcpyAsync(P.p[k], A.given[k], (size_t)g.stride[k] * (k ? g.height >> 1 : g.height) * 2, cudaMemcpyDeviceToDevice, s));
  }
  // 1. K2 inter prediction
  if (A.numPus) {
    McLaunch L; L.geom = g; L.dst = P; memset(L.refs, 0, sizeof(L.refs));
    for (int sl = 0; sl < c->numSlots; sl++) { DevPlanes d = c->planes(c->slotBuf[sl]); for (int k = 0; k < 3; k++) L.refs[sl * 3 + k] = d.p[k]; }
    for (int k = 0; k < 3; k++) L.refStride[k] = g.stride[k];
    L.pus = A.pus; L.tiles = A.tiles; L.meta = A.mcMeta; L.dmvrMv = A.dmvrMv; L.lmcs = A.lmcs; L.wp = A.wp;
    for (int l = 0; l < MC_LISTS; l++) L.cnt[l] = A.hMeta[LM_CNT + l];
    if (int rc = launch_mc(L, c->ss, c->profiling ? &c->prof : nullptr)) return rc;
    c->launches += mc_launch_count(L);
  }
  // 2. K1 residual + reco, 2b. K6 intra blocks in decoding order (prediction from the reconstruction so far — inter CUs, earlier intra blocks — + their
  // residual).  With LMCS chroma scaling the chroma residual scale of a VPDU is derived from its reconstructed (mapped-domain) luma neighbourhood
  // (Reshape.cpp:192), intra blocks included: luma TUs -> luma intra blocks -> per-VPDU scale -> chroma TUs (scaled) -> chroma intra blocks.
  LmcsLaunch LM; LM.geom = g; LM.planes = P; LM.lmcs = A.lmcs; LM.vpdus = A.lmcsVpdus; LM.invLut = A.lmcsInv; LM.scale = A.lmcsScale;
  const bool twoPass = A.lmcs && A.lmcsChromaAdj;
  A.hMeta[2 * LM_INTS] = 0;
  int16_t* resiPl[3] = {nullptr, nullptr, nullptr};
  if (A.numIntraTus) {
    uint8_t* rb = c->resiBuf.as<uint8_t>(); resiPl[0] = reinterpret_cast<int16_t*>(rb); resiPl[1] = reinterpret_cast<int16_t*>(rb + c->planeBytes[0]); resiPl[2] = reinterpret_cast<int16_t*>(rb + c->planeBytes[0] + c->planeBytes[1]);
    if (A.ciipResi) { if (int rc = launch_intra_ciip_clear(A.intraTus, A.numIntraTus, resiPl, P.stride, s)) return rc; c->launches += 1; }
  }
  auto runK1 = [&](int compSel, const int* vpduScale) -> int {
    if (!A.numTus) return 0;
    K1Launch L; L.geom = g; L.planes = P; L.tus = A.tus; L.numTus = A.numTus; L.idx = A.tuIdx; L.meta = A.tuMeta; L.coefs = A.coefs; L.scaling = A.scaling; L.mode = 0;
    for (int k = 0; k < 3; k++) L.resi[k] = resiPl[k];
    for (int l = 0; l < K1_LISTS; l++) L.cnt[l] = A.hMeta[LM_INTS + LM_CNT + l];
    L.compSel = compSel; L.vpduScale = vpduScale;
    if (int rc = launch_k1_residual(L, c->ss, c->profiling ? &c->prof : nullptr)) return rc;
    c->launches += k1_launch_count(L);
    return 0;
  };
  auto runK6 = [&](int compSel) -> int {
    if (!A.numIntraTus) return 0;
    IntraLaunch L; L.geom = g; L.planes = P; L.tus = A.intraTus; L.numTus = A.numIntraTus; L.sync = A.intraSync; L.order = A.intraOrder; L.compSel = compSel;
    for (int k = 0; k < 3; k++) { L.resi[k] = resiPl[k]; L.owner[k] = A.intraOwner[k]; L.ownerStride[k] = A.intraOwnerStride[k]; L.ownerBytes[k] = A.intraOwnerBytes[k]; }
    if (c->profiling) c->prof.begin(B200_KF_INTRA, s);
    if (int rc = launch_intra(L, s)) return rc;
    if (c->profiling) c->prof.end(B200_KF_INTRA, s);
    c->launches += compSel == 2 ? 1 : 5;
    return 0;
  };
  if (twoPass) {
    if (int rc = runK1(1, nullptr)) return rc;
    if (int rc = runK6(1)) return rc;
    if (c->profiling) c->prof.begin(B200_KF_LMCS, s);
    if (int rc = launch_lmcs_vpdu(LM, s)) return rc;
    if (c->profiling) c->prof.end(B200_KF_LMCS, s);
    c->launches += 1;
    if (int rc = runK1(2, A.lmcsScale)) return rc;
    if (int rc = runK6(2)) return rc;
  } else {
    if (int rc = runK1(0, nullptr)) return rc;
    if (int rc = runK6(0)) return rc;
  }
  if (A.numIntraTus) B200_CUDA(cudaMemcpyAsync(A.hMeta + 2 * LM_INTS, A.intraSync + A.numIntraTus + 1, sizeof(int), cudaMemcpyDeviceToHost, s));   // timeout bit, read by b200_wait_picture
  if (A.lmcs) { if (c->profiling) c->prof.begin(B200_KF_LMCS, s); if (int rc = launch_lmcs_inv(LM, s)) return rc; if (c->profiling) c->prof.end(B200_KF_LMCS, s); c->launches += 1; }   // RSP stage (DecLibRecon.cpp:935)
  // 3. K3 deblocking
  if (A.flags & B200_PIC_DEBLOCK) {
    LfLaunch L; L.geom = g; L.planes = P; L.lfV = A.lfV; L.lfH = A.lfH; L.ctuSlice = A.ctuSlice; L.slices = A.lfSlices; L.seq = A.lfSeq; L.dirs = 3;
    if (int rc = launch_lf_deblock(L, s, c->profiling ? &c->prof : nullptr)) return rc;
    c->launches += 2;
  }
  // 4. K4 SAO (out of place)
  if (A.flags & B200_PIC_SAO) {
    SaoLaunch L; L.geom = g; L.src = P; L.dst = c->planes(other); L.ctus = A.sao; L.vb = A.vb;
    if (int rc = launch_sao(L, s, c->profiling ? &c->prof : nullptr)) return rc;
    c->launches += 1;
    std::swap(cur, other); P = c->planes(cur);
  }
  // 5. K5 ALF (out of place, straight into a buffer that becomes the DPB slot)
  if (A.flags & B200_PIC_ALF) {
    AlfLaunch L; L.geom = g; L.src = P; L.dst = c->planes(other); L.ctus = A.alf;
    L.lumaCoeff = A.lumaCoeff; L.lumaClip = A.lumaClip; L.chromaCoeff = A.chromaCoeff; L.chromaClip = A.chromaClip; L.cc[0] = A.cc[0]; L.cc[1] = A.cc[1];
    if (int rc = launch_alf(L, c->ss, c->profiling ? &c->prof : nullptr)) return rc;
    c->launches += g.chromaFormat ? 2 : 1;
    std::swap(cur, other);
  }
  B200_CUDA(cudaEventRecord(A.done, s)); A.donePending = true;
  // 6. the buffer holding the result becomes the slot's buffer; the slot's old buffer becomes a work buffer (swapBufs, DecLibRecon.cpp:423)
  const int old = c->slotBuf[A.dstSlot];
  c->slotBuf[A.dstSlot] = cur;
  c->work[0] = old; c->work[1] = other;
  return 0;
}

B200_API int b200_decompress_picture(b200_ctx* c, const b200_picture* p)
{
  const int ai = b200_pic_upload(c, p);
  if (ai < 0) return ai;
  if (int rc = b200_pic_run(c, ai)) return rc;
  return ai;
}

B200_API int b200_wait_picture(b200_ctx* c, int ai, int32_t* dmvrMv, size_t numDmvr)
{
  B200_CHECK(c, "b200_wait_picture: null context");
  if (dmvrMv && ai >= 0 && ai < c->numArenas && c->arenas[ai].dmvrMv) {
    const size_t n = numDmvr < c->arenas[ai].numDmvr ? numDmvr : c->arenas[ai].numDmvr;
    if (n) { if (int rc = copy_host(dmvrMv, c->arenas[ai].dmvrMv, n * 8, cudaMemcpyDeviceToHost, c->stream)) return rc; }
  }
  B200_CUDA(cudaStreamSynchronize(c->upStream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  if (ai >= 0 && ai < c->numArenas && c->arenas[ai].numIntraTus) {
    const int err = c->arenas[ai].hMeta[2 * LM_INTS];
    B200_CHECK(!(err & INTRA_ERR_CTU_BLOCKS), "b200_wait_picture: a CTU holds more than %d intra block records (overlapping records?)", INTRA_MAX_CTU_BLOCKS);
    B200_CHECK(!err, "b200_wait_picture: an intra block waited for a neighbour that never finished (intra list not in decoding order?)");
  }
  return 0;
}

B200_API int b200_get_frame(b200_ctx* c, int slot, int16_t* const planes[3])
{
  B200_CHECK(c && planes && slot >= 0 && slot < c->numSlots, "b200_get_frame: bad argument");
  DevPlanes d = c->planes(c->slotBuf[slot]);
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++)
    if (int rc = copy_host(planes[k], d.p[k], (size_t)c->g.stride[k] * (k ? c->g.height >> 1 : c->g.height) * 2, cudaMemcpyDeviceToHost, c->stream)) return rc;
  B200_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

// Picture buffers of the host decoder carry margins (stride > width): 2-D copies between the margin-less device planes and strided host planes.
// The runtime classifies a host range by its first address.  cudaHostRegister pins whole pages, so a plane that starts on a page the caller registered for
// another array (the glue pins its work-list vectors, which share the heap with the decoder's picture buffers) and runs past that registration is refused with
// cudaErrorInvalidValue.  Such a plane, like any other caller array this file copies (copy_host), goes through a pinned staging copy instead.
static int copy2d_host(void* dst, size_t dpitch, const void* src, size_t spitch, size_t wBytes, size_t h, cudaMemcpyKind kind, cudaStream_t s)
{
  const cudaError_t e = cudaMemcpy2DAsync(dst, dpitch, src, spitch, wBytes, h, kind, s);
  if (e != cudaErrorInvalidValue) { B200_CUDA(e); return 0; }
  (void)cudaGetLastError();
  void* stage = nullptr;
  B200_CUDA(cudaMallocHost(&stage, wBytes * h));
  int rc = 0;
  if (kind == cudaMemcpyHostToDevice) {
    for (size_t y = 0; y < h; y++) memcpy((char*)stage + y * wBytes, (const char*)src + y * spitch, wBytes);
    const cudaError_t e2 = cudaMemcpy2DAsync(dst, dpitch, stage, wBytes, wBytes, h, kind, s);
    const cudaError_t e3 = e2 == cudaSuccess ? cudaStreamSynchronize(s) : e2;
    if (e3 != cudaSuccess) { set_error("copy2d_host: staged H2D copy -> %s", cudaGetErrorString(e3)); (void)cudaGetLastError(); rc = B200_ERR_CUDA; }
  } else {
    const cudaError_t e2 = cudaMemcpy2DAsync(stage, wBytes, src, spitch, wBytes, h, kind, s);
    const cudaError_t e3 = e2 == cudaSuccess ? cudaStreamSynchronize(s) : e2;
    if (e3 != cudaSuccess) { set_error("copy2d_host: staged D2H copy -> %s", cudaGetErrorString(e3)); (void)cudaGetLastError(); rc = B200_ERR_CUDA; }
    else for (size_t y = 0; y < h; y++) memcpy((char*)dst + y * dpitch, (const char*)stage + y * wBytes, wBytes);
  }
  cudaFreeHost(stage);
  return rc;
}

B200_API int b200_ctx_load_slot_strided(b200_ctx* c, int slot, const int16_t* const planes[3], const ptrdiff_t strides[3])
{
  B200_CHECK(c && planes && strides && slot >= 0 && slot < c->numSlots, "b200_ctx_load_slot_strided: bad argument");
  if (int rc = wait_readers(c, c->slotBuf[slot])) return rc;
  DevPlanes d = c->planes(c->slotBuf[slot]);
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++) {
    const size_t w = k ? c->g.width >> 1 : c->g.width, h = k ? c->g.height >> 1 : c->g.height;
    B200_CHECK(planes[k] && strides[k] >= (ptrdiff_t)w, "b200_ctx_load_slot_strided: plane %d", k);
    if (int rc = copy2d_host(d.p[k], (size_t)c->g.stride[k] * 2, planes[k], (size_t)strides[k] * 2, w * 2, h, cudaMemcpyHostToDevice, c->stream)) return rc;
  }
  B200_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

B200_API int b200_get_frame_strided(b200_ctx* c, int slot, int16_t* const planes[3], const ptrdiff_t strides[3])
{
  B200_CHECK(c && planes && strides && slot >= 0 && slot < c->numSlots, "b200_get_frame_strided: bad argument");
  DevPlanes d = c->planes(c->slotBuf[slot]);
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++) {
    const size_t w = k ? c->g.width >> 1 : c->g.width, h = k ? c->g.height >> 1 : c->g.height;
    B200_CHECK(planes[k] && strides[k] >= (ptrdiff_t)w, "b200_get_frame_strided: plane %d", k);
    if (int rc = copy2d_host(planes[k], (size_t)strides[k] * 2, d.p[k], (size_t)c->g.stride[k] * 2, w * 2, h, cudaMemcpyDeviceToHost, c->stream)) return rc;
  }
  B200_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

B200_API int b200_get_frame_async(b200_ctx* c, int slot, int16_t* const planes[3])
{
  B200_CHECK(c && planes && slot >= 0 && slot < c->numSlots, "b200_get_frame_async: bad argument");
  const int buf = c->slotBuf[slot];
  DevPlanes d = c->planes(buf);
  B200_CUDA(cudaEventRecord(c->finalEv, c->stream));                 // everything submitted so far (incl. this slot's picture) is final after this
  B200_CUDA(cudaStreamWaitEvent(c->copyStream, c->finalEv, 0));
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++)
    if (int rc = copy_host(planes[k], d.p[k], (size_t)c->g.stride[k] * (k ? c->g.height >> 1 : c->g.height) * 2, cudaMemcpyDeviceToHost, c->copyStream)) return rc;
  if (int rc = mark_read(c, buf, c->copyStream)) return rc;
  const int t = c->nextTicket; c->nextTicket = (c->nextTicket + 1) & 15;
  B200_CUDA(cudaEventRecord(c->ticketEv[t], c->copyStream));
  return t;
}

// Device-to-device output on a stream of the caller's (multi-GPU gather: the frame goes to a send buffer, NCCL takes it from there): the caller's stream
// waits for everything submitted so far, the copies run on it, and later pictures wait for them before they overwrite the DPB buffer.
B200_API int b200_get_frame_device_async(b200_ctx* c, int slot, int16_t* const planesDev[3], void* cudaStream)
{
  B200_CHECK(c && planesDev && slot >= 0 && slot < c->numSlots, "b200_get_frame_device_async: bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(cudaStream);
  const int buf = c->slotBuf[slot];
  DevPlanes d = c->planes(buf);
  B200_CUDA(cudaEventRecord(c->finalEv, c->stream));
  B200_CUDA(cudaStreamWaitEvent(st, c->finalEv, 0));
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++) {
    B200_CHECK(planesDev[k], "b200_get_frame_device_async: plane %d", k);
    B200_CUDA(cudaMemcpyAsync(planesDev[k], d.p[k], (size_t)c->g.stride[k] * (k ? c->g.height >> 1 : c->g.height) * 2, cudaMemcpyDeviceToDevice, st));
  }
  if (int rc = mark_read(c, buf, st)) return rc;
  return 0;
}

B200_API size_t b200_frame_bytes(const b200_geom* g, int fmt, int comp)
{
  if (!g || comp < 0 || comp > 2 || (comp && !g->chromaFormat)) return 0;
  const size_t W = comp ? g->width >> 1 : g->width, H = comp ? g->height >> 1 : g->height;
  if (fmt == B200_OUT_PYUV) return W / 4 * 5 * H;
  if (fmt == B200_OUT_8) return W * H;
  return (size_t)g->stride[comp] * H * 2;
}

B200_API int b200_get_frame_fmt_async(b200_ctx* c, int slot, int fmt, void* const planes[3])
{
  B200_CHECK(c && planes && slot >= 0 && slot < c->numSlots, "b200_get_frame_fmt_async: bad argument");
  if (fmt == B200_OUT_16) { int16_t* const p16[3] = {(int16_t*)planes[0], (int16_t*)planes[1], (int16_t*)planes[2]}; return b200_get_frame_async(c, slot, p16); }
  B200_CHECK(fmt == B200_OUT_PYUV || fmt == B200_OUT_8, "b200_get_frame_fmt_async: unknown format %d", fmt);
  if (fmt == B200_OUT_PYUV && (c->g.bitDepth != 10 || (c->g.width & 7))) { set_error("b200_get_frame_fmt_async: pyuv needs 10 bit and a width divisible by 8 (as vvdecapp)"); return B200_ERR_UNSUPPORTED; }
  B200_CUDA(cudaSetDevice(c->device));
  const int nPl = c->g.chromaFormat ? 3 : 1;
  size_t bytes[3] = {0, 0, 0}, off[3] = {0, 0, 0}, total = 0;
  for (int k = 0; k < nPl; k++) { bytes[k] = b200_frame_bytes(&c->g, fmt, k); off[k] = total; total += (bytes[k] + 255) & ~(size_t)255; }
  const int st = c->nextStage; c->nextStage ^= 1;
  if (total > c->outStage[st].cap) B200_CUDA(cudaStreamSynchronize(c->copyStream));          // growing: no copy may still read the old block
  if (int rc = c->outStage[st].reserve(total)) return rc;
  const int buf = c->slotBuf[slot];
  DevPlanes d = c->planes(buf);
  B200_CUDA(cudaEventRecord(c->finalEv, c->stream));
  B200_CUDA(cudaStreamWaitEvent(c->copyStream, c->finalEv, 0));
  uint8_t* dst[3]; for (int k = 0; k < 3; k++) dst[k] = c->outStage[st].as<uint8_t>() + off[k];
  if (int rc = launch_pack(d, c->g, fmt, dst, c->copyStream)) return rc;                      // on the copy stream: the kernel stream runs on
  c->launches += nPl;
  if (int rc = mark_read(c, buf, c->copyStream)) return rc;                                   // the picture buffer is free once it is packed
  for (int k = 0; k < nPl; k++) if (int rc = copy_host(planes[k], dst[k], bytes[k], cudaMemcpyDeviceToHost, c->copyStream)) return rc;
  const int t = c->nextTicket; c->nextTicket = (c->nextTicket + 1) & 15;
  B200_CUDA(cudaEventRecord(c->ticketEv[t], c->copyStream));
  return t;
}

B200_API int b200_get_frame_grain_async(b200_ctx* c, int slot, int fmt, void* const planes[3], const b200_film_grain* fg)
{
  B200_CHECK(c && planes && fg && slot >= 0 && slot < c->numSlots, "b200_get_frame_grain_async: bad argument");
  B200_CHECK(fg->pattern && fg->sLUT && fg->pLUT && fg->lineSeeds, "b200_get_frame_grain_async: table missing");
  B200_CHECK(fmt == B200_OUT_16 || fmt == B200_OUT_PYUV || fmt == B200_OUT_8, "b200_get_frame_grain_async: unknown format %d", fmt);
  const b200_geom& g = c->g;
  if (g.bitDepth != 8 && g.bitDepth != 10) { set_error("b200_get_frame_grain_async: film grain needs 8 or 10 bit (FilmGrainImpl::set_depth)"); return B200_ERR_UNSUPPORTED; }
  if (fmt == B200_OUT_PYUV && (g.bitDepth != 10 || (g.width & 7))) { set_error("b200_get_frame_grain_async: pyuv needs 10 bit and a width divisible by 8 (as vvdecapp)"); return B200_ERR_UNSUPPORTED; }
  const int bs = g.bitDepth - 8;
  B200_CHECK(fg->scaleShift + bs >= 8 && fg->scaleShift + bs <= 13, "b200_get_frame_grain_async: scaleShift %d out of range (FilmGrainImpl.cpp:142)", fg->scaleShift);
  B200_CHECK(g.width > 128, "b200_get_frame_grain_async: width must exceed 128 (FilmGrainImpl.cpp:140)");
  for (int k = 0; k < 768; k++) B200_CHECK((fg->pLUT[k] >> 4) < 8, "b200_get_frame_grain_async: pLUT[%d] selects pattern %d (only 8 exist)", k, fg->pLUT[k] >> 4);
  B200_CUDA(cudaSetDevice(c->device));
  const int nPl = g.chromaFormat ? 3 : 1, nbx = (g.width + 15) / 16, nby = (g.height + 15) / 16;
  const int st = c->nextStage; c->nextStage ^= 1;
  // device copies of the tables: [pattern 64 KB][sLUT][pLUT][line seeds][block seeds]; every use is ordered on the copy stream
  const size_t oS = 2 * 8 * 4096, oP = oS + 768, oL = oP + 768, oB = oL + (size_t)nby * 4, tabBytes = oB + (size_t)nbx * nby * 4;
  if (tabBytes > c->grainTab.cap || c->picBytes > c->grainStage[st].cap) B200_CUDA(cudaStreamSynchronize(c->copyStream));   // growing: nothing may still use the old block
  if (int rc = c->grainTab.reserve(tabBytes)) return rc;
  if (int rc = c->grainStage[st].reserve(c->picBytes)) return rc;
  uint8_t* tb = c->grainTab.as<uint8_t>();
  // The caller may reuse its arrays once this call returns, while the H2D copy may still wait behind earlier work of the copy stream: the tables go through
  // pinned memory of the context first.  Stage st is refilled once the copy of the call before last that used it has run.
  auto& hs = c->grainHost[st];
  if (hs.pending) { B200_CUDA(cudaEventSynchronize(hs.copied)); hs.pending = false; }
  if (oB > hs.cap) {
    if (hs.p) cudaFreeHost(hs.p);
    hs.p = nullptr; hs.cap = 0;
    B200_CUDA(cudaHostAlloc(&hs.p, oB, cudaHostAllocDefault)); hs.cap = oB;
  }
  uint8_t* hb = static_cast<uint8_t*>(hs.p);
  memcpy(hb, fg->pattern, oS); memcpy(hb + oS, fg->sLUT, 768); memcpy(hb + oP, fg->pLUT, 768); memcpy(hb + oL, fg->lineSeeds, (size_t)nby * 4);
  B200_CUDA(cudaMemcpyAsync(tb, hb, oB, cudaMemcpyHostToDevice, c->copyStream));
  B200_CUDA(cudaEventRecord(hs.copied, c->copyStream)); hs.pending = true;
  const int buf = c->slotBuf[slot];
  DevPlanes src = c->planes(buf), gr = src;
  { uint8_t* b = c->grainStage[st].as<uint8_t>(); gr.p[0] = reinterpret_cast<int16_t*>(b); gr.p[1] = reinterpret_cast<int16_t*>(b + c->planeBytes[0]); gr.p[2] = reinterpret_cast<int16_t*>(b + c->planeBytes[0] + c->planeBytes[1]); }
  B200_CUDA(cudaEventRecord(c->finalEv, c->stream));
  B200_CUDA(cudaStreamWaitEvent(c->copyStream, c->finalEv, 0));
  if (int rc = launch_film_grain(src, gr, g, reinterpret_cast<const int8_t*>(tb), tb + oS, tb + oP, reinterpret_cast<const uint32_t*>(tb + oL),
                                 reinterpret_cast<uint32_t*>(tb + oB), fg->scaleShift, fg->compPresent, c->copyStream)) return rc;
  c->launches += 1 + nPl;
  if (int rc = mark_read(c, buf, c->copyStream)) return rc;                                   // the picture buffer is free once the grained copy exists
  if (fmt == B200_OUT_16) {
    for (int k = 0; k < nPl; k++) if (int rc = copy_host(planes[k], gr.p[k], (size_t)g.stride[k] * (k ? g.height >> 1 : g.height) * 2, cudaMemcpyDeviceToHost, c->copyStream)) return rc;
  } else {
    size_t bytes[3] = {0, 0, 0}, off[3] = {0, 0, 0}, total = 0;
    for (int k = 0; k < nPl; k++) { bytes[k] = b200_frame_bytes(&g, fmt, k); off[k] = total; total += (bytes[k] + 255) & ~(size_t)255; }
    if (total > c->outStage[st].cap) B200_CUDA(cudaStreamSynchronize(c->copyStream));
    if (int rc = c->outStage[st].reserve(total)) return rc;
    uint8_t* dst[3]; for (int k = 0; k < 3; k++) dst[k] = c->outStage[st].as<uint8_t>() + off[k];
    if (int rc = launch_pack(gr, g, fmt, dst, c->copyStream)) return rc;
    c->launches += nPl;
    for (int k = 0; k < nPl; k++) if (int rc = copy_host(planes[k], dst[k], bytes[k], cudaMemcpyDeviceToHost, c->copyStream)) return rc;
  }
  const int t = c->nextTicket; c->nextTicket = (c->nextTicket + 1) & 15;
  B200_CUDA(cudaEventRecord(c->ticketEv[t], c->copyStream));
  return t;
}

B200_API int b200_frame_hash_async(b200_ctx* c, int slot, int method, uint8_t* digest)
{
  B200_CHECK(c && digest && slot >= 0 && slot < c->numSlots, "b200_frame_hash_async: bad argument");
  if (method == B200_HASH_MD5) { set_error("b200_frame_hash_async: MD5 is a serial chain over each plane and is not computed on the device; use CRC or checksum"); return B200_ERR_UNSUPPORTED; }
  B200_CHECK(method == B200_HASH_CRC || method == B200_HASH_CHECKSUM, "b200_frame_hash_async: unknown method %d", method);
  B200_CUDA(cudaSetDevice(c->device));
  if (int rc = c->hashBuf.reserve(16 * 32)) return rc;                                        // per ticket: 3 accumulators + 12 digest bytes
  const int t = c->nextTicket; c->nextTicket = (c->nextTicket + 1) & 15;
  uint32_t* acc = c->hashBuf.as<uint32_t>() + t * 8; uint8_t* dig = reinterpret_cast<uint8_t*>(acc + 4);
  const int buf = c->slotBuf[slot];
  B200_CUDA(cudaEventRecord(c->finalEv, c->stream));
  B200_CUDA(cudaStreamWaitEvent(c->copyStream, c->finalEv, 0));
  B200_CUDA(cudaMemsetAsync(acc, 0, 32, c->copyStream));
  if (int rc = launch_hash(c->planes(buf), c->g, method, acc, dig, c->copyStream)) return rc;
  c->launches += (c->g.chromaFormat ? 3 : 1) + 1;
  if (int rc = mark_read(c, buf, c->copyStream)) return rc;
  if (int rc = copy_host(digest, dig, 12, cudaMemcpyDeviceToHost, c->copyStream)) return rc;
  B200_CUDA(cudaEventRecord(c->ticketEv[t], c->copyStream));
  return t;
}

B200_API int b200_frame_wait(b200_ctx* c, int ticket)
{
  B200_CHECK(c && ticket >= 0 && ticket < 16, "b200_frame_wait: bad ticket");
  B200_CUDA(cudaEventSynchronize(c->ticketEv[ticket]));
  return 0;
}

B200_API int b200_ctx_mark(b200_ctx* c, int which) { B200_CHECK(c && (which == 0 || which == 1), "b200_ctx_mark"); B200_CUDA(cudaEventRecord(c->ev[which], c->stream)); return 0; }
B200_API int b200_ctx_elapsed_ms(b200_ctx* c, float* ms) { B200_CHECK(c && ms, "b200_ctx_elapsed_ms"); B200_CUDA(cudaEventSynchronize(c->ev[1])); B200_CUDA(cudaEventElapsedTime(ms, c->ev[0], c->ev[1])); return 0; }
B200_API long long b200_ctx_kernel_launches(b200_ctx* c) { return c ? c->launches : 0; }

B200_API int b200_ctx_set_profiling(b200_ctx* c, int on) { B200_CHECK(c, "b200_ctx_set_profiling"); c->profiling = on != 0; return 0; }

B200_API int b200_ctx_get_kernel_ms_n(b200_ctx* c, float* ms, int* counts, int n)
{
  B200_CHECK(c && ms && counts && n >= 1 && n <= B200_KF_COUNT, "b200_ctx_get_kernel_ms_n");
  B200_CUDA(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < n; i++) { ms[i] = 0; counts[i] = 0; }
  for (auto& r : c->prof.recs) { float t = 0; cudaEventElapsedTime(&t, r.a, r.b); if (r.family < n) { ms[r.family] += t; counts[r.family]++; } c->prof.pool.push_back(r.a); c->prof.pool.push_back(r.b); }
  c->prof.recs.clear();
  return 0;
}
B200_API int b200_ctx_get_kernel_ms(b200_ctx* c, float ms[8], int counts[8]) { return b200_ctx_get_kernel_ms_n(c, ms, counts, 8); }

B200_API int b200_host_register(void* ptr, size_t bytes) { B200_CHECK(ptr && bytes, "b200_host_register"); if (int rc = ensure_device()) return rc; B200_CUDA(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault)); return 0; }
B200_API int b200_host_unregister(void* ptr) { B200_CHECK(ptr, "b200_host_unregister"); B200_CUDA(cudaHostUnregister(ptr)); return 0; }

}  // extern "C"
