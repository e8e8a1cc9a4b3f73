// picture.cu — picture-level context: device-resident DPB, work-list arenas, and the per-picture kernel chain
// (the device replacement of DecLibRecon::decompressPicture's CTU task graph, reference DecoderLib/DecLibRecon.cpp:429-682).
#include "common.cuh"
#include "lf_derive.cuh"
#include <string.h>
#include <vector>

namespace b200 {

struct Arena {
  DevBuf buf;                       // one allocation, sub-allocated per picture
  // The launch records of the picture's kernels, filled by b200_pic_upload.  b200_pic_run adds what is known at run time: planes, reference slots,
  // list counts (hMeta) and compSel.
  McLaunch mc; K1Launch k1; IntraLaunch intra; LmcsLaunch lm; LfLaunch lf; SaoLaunch sao; AlfLaunch alf; LfDeriveLaunch lfd;
  int* hMeta = nullptr;             // pinned host copy of both meta blocks (list lengths + error bits), valid once `uploaded` has fired
  size_t numPus = 0, numDmvr = 0;
  DevPlanes given;                  // pre-reconstructed samples, or null planes
  int dstSlot = 0, flags = 0;
  bool lmcsChromaAdj = false;
  bool ciipResi = false;             // a CIIP block takes a residual: its residual-plane area is cleared before K1 (k6_intra.cu)
  bool valid = false;
  cudaEvent_t uploaded = nullptr, done = nullptr; bool donePending = false;   // H2D finished / kernels reading this arena finished
};

// Picture buffers of the host decoder carry margins (stride > width): 2-D copies between the margin-less device planes and strided host planes.
// The runtime classifies a host range by its first address.  cudaHostRegister pins whole pages, so a plane that starts on a page the caller registered for
// another array (the glue pins its work-list vectors, which share the heap with the decoder's picture buffers) and runs past that registration is refused with
// cudaErrorInvalidValue.  Such a plane, like any other caller array this file copies (copy_host), goes through a pinned staging copy instead.
int copy2d_host(void* dst, size_t dpitch, const void* src, size_t spitch, size_t wBytes, size_t h, cudaMemcpyKind kind, cudaStream_t s)
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

int Staging::commit(DevBuf& buf, cudaStream_t s)
{
  if (int rc = buf.reserve(bytes())) return rc;
  char* base = buf.as<char>();
  for (const Part& q : parts) q.set(q.view, q.span ? base + q.off : nullptr);
  for (const Part& q : parts) if (q.copy) if (int rc = copy_host(base + q.off, q.src, q.copy, cudaMemcpyHostToDevice, s)) return rc;
  return 0;
}

}  // namespace b200

using namespace b200;

// The context's launch hook: counts every kernel the context issues and, while profiling is on, records an event pair per launcher call and family.
struct CtxHook : b200::KHook {
  struct Rec { int family; cudaEvent_t a, b; };
  std::vector<Rec> recs; std::vector<cudaEvent_t> pool; Rec cur{}; bool profiling = false;
  cudaEvent_t get() { cudaEvent_t e; if (!pool.empty()) { e = pool.back(); pool.pop_back(); } else cudaEventCreate(&e); return e; }
  void begin(int f, cudaStream_t s) override { if (!profiling) return; cur.family = f; cur.a = get(); cur.b = get(); cudaEventRecord(cur.a, s); }
  void end(int, cudaStream_t s) override { if (!profiling) return; cudaEventRecord(cur.b, s); recs.push_back(cur); }
};

struct b200_ctx {
  b200_geom g;
  CtxHook hook;
  int numSlots = 0, numArenas = 0, device = 0;
  cudaStream_t stream = nullptr, copyStream = nullptr, upStream = nullptr;   // kernels / frame output D2H / work-list H2D
  StreamSet ss;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  std::vector<cudaEvent_t> readDone; std::vector<char> readPending;   // per picture buffer: an async output (maybe) still reads it (mark_read)
  std::vector<cudaStream_t> readStream;                              // the stream readDone was last recorded on
  cudaEvent_t ticketEv[16]; cudaEvent_t finalEv = nullptr; int nextTicket = 0;
  DevBuf outStage[2]; int nextStage = 0;   // converted output frames (pyuv / 8 bit) waiting for their D2H copy
  size_t picBytes = 0;
  std::vector<int16_t*> bufs;          // numSlots + 2 picture buffers
  std::vector<int> slotBuf;            // slot -> buffer index
  int work[2] = {0, 0};                // indices of the two work buffers
  std::vector<Arena> arenas;
  int nextArena = 0;
  DevBuf grainStage[2], grainTab;    // b200_get_frame_grain_async: grained copy of the frame, device copies of the tables + block seeds
  struct HostStage { void* p = nullptr; size_t cap = 0; cudaEvent_t copied = nullptr; bool pending = false; } grainHost[2];   // pinned copies of the caller's tables
  DevBuf resiBuf;                    // residual planes of intra CUs (K1 -> K6), allocated with the first picture that carries intra blocks
  DevBuf hashBuf;                    // b200_frame_hash_async: accumulators + digest per ticket

  DevPlanes planes(int buf) const { return pic_planes(bufs[buf], g); }
};

extern "C" {

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
  c->picBytes = pic_bytes(*g);
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

// The synchronous copies between a slot's buffer and caller planes: whole strides, padding included (strides null), or plane widths at the caller's strides
static int copy_slot(b200_ctx* c, int slot, int16_t* const host[3], const ptrdiff_t* strides, cudaMemcpyKind kind, const char* fn)
{
  const b200_geom& g = c->g;
  if (kind == cudaMemcpyHostToDevice) if (int rc = wait_readers(c, c->slotBuf[slot])) return rc;
  DevPlanes d = c->planes(c->slotBuf[slot]);
  for (int k = 0; k < (g.chromaFormat ? 3 : 1); k++) {
    const size_t w = k ? g.width >> 1 : g.width, h = k ? g.height >> 1 : g.height;
    if (strides) B200_CHECK(host[k] && strides[k] >= (ptrdiff_t)w, "%s: plane %d", fn, k);
    const size_t dp = strides ? (size_t)g.stride[k] * 2 : plane_bytes(g, k), hp = strides ? (size_t)strides[k] * 2 : dp, wb = strides ? w * 2 : dp;
    const int rc = kind == cudaMemcpyHostToDevice ? copy2d_host(d.p[k], dp, host[k], hp, wb, strides ? h : 1, kind, c->stream)
                                                  : copy2d_host(host[k], hp, d.p[k], dp, wb, strides ? h : 1, kind, c->stream);
    if (rc) return rc;
  }
  B200_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

B200_API int b200_ctx_load_slot(b200_ctx* c, int slot, const int16_t* const planes[3])
{
  B200_CHECK(c && planes && slot >= 0 && slot < c->numSlots, "b200_ctx_load_slot: bad argument");
  return copy_slot(c, slot, const_cast<int16_t* const*>(planes), nullptr, cudaMemcpyHostToDevice, "b200_ctx_load_slot");
}

B200_API int b200_pic_upload(b200_ctx* c, const b200_picture* p)
{
  B200_CHECK(c && p, "b200_pic_upload: null argument");
  B200_CHECK(p->dstSlot >= 0 && p->dstSlot < c->numSlots, "b200_pic_upload: dstSlot %d", p->dstSlot);
  const bool lfd = p->flags & B200_PIC_DERIVE_LF;
  B200_CHECK(!lfd || ((p->flags & B200_PIC_DEBLOCK) && !p->lfV && !p->lfH && p->lfCus && p->numLfCus && p->lfTus && p->lfCtuCus && p->lfSliceB && p->numLfCus < (1u << 31) && p->numLfTus < (1u << 31)),
             "b200_pic_upload: B200_PIC_DERIVE_LF needs B200_PIC_DEBLOCK, CU / TU records, CTU ranges and slice types, and no lfV / lfH");
  B200_CHECK(!(p->flags & B200_PIC_DEBLOCK) || ((lfd || (p->lfV && p->lfH)) && p->lfSlices && p->numLfSlices >= 1 && p->numLfSlices <= 64), "b200_pic_upload: deblocking data missing");
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
  const int vs = g.ctuSize == 128 ? 64 : g.ctuSize; const size_t nVpdu = (size_t)((g.width + vs - 1) / vs) * ((g.height + vs - 1) / vs);
  const bool lf = p->flags & B200_PIC_DEBLOCK, sao = p->flags & B200_PIC_SAO, alf = p->flags & B200_PIC_ALF, lm = p->flags & B200_PIC_LMCS, given = p->given[0];
  const size_t capTiles = mc_tile_capacity(g, 0), ni = p->numIntraTus;
  A.mc.geom = A.k1.geom = A.intra.geom = A.lm.geom = A.lf.geom = A.sao.geom = A.alf.geom = g;
  intra_owner_maps(A.intra);
  // No per-record work on the host: the caller's arrays are copied as they are; the records are validated and sorted into the
  // kernels' work lists on the device (bucket.cu), errors surface in b200_pic_run.
  uint32_t *tiles, *tuIdx; int* meta;
  Staging st;
  st.add(&A.mc.pus, p->pus, p->numPus); st.add(&tiles, nullptr, capTiles); st.add(&meta, nullptr, 2 * LM_INTS); st.add(&tuIdx, nullptr, p->numTus);
  st.add(&A.k1.tus, p->tus, p->numTus); st.add(&A.k1.coefs, p->coefs, p->numCoefs); st.add(&A.k1.scaling, p->scaling, p->numScaling);
  st.add(&A.lf.lfV, lfd ? nullptr : p->lfV, lf ? n4 : 0); st.add(&A.lf.lfH, lfd ? nullptr : p->lfH, lf ? n4 : 0);
  if (lfd) {                                                          // (the arena of a picture without it keeps its layout)
    st.add(&A.lfd.cus, p->lfCus, p->numLfCus); st.add(&A.lfd.tus, p->lfTus, p->numLfTus); st.add(&A.lfd.ctuCus, p->lfCtuCus, nCtu + 1);
    st.add(&A.lfd.sliceB, p->lfSliceB, (size_t)p->numLfSlices); st.add(&A.lfd.slices, p->lfSlices, (size_t)p->numLfSlices);
    st.add(&A.lfd.map[0], nullptr, 2 * n4); st.add(&A.lfd.mi, nullptr, n4);
  }
  st.add(&A.lf.ctuSlice, lf ? p->ctuSlice : nullptr, nCtu);
  st.add(&A.sao.ctus, p->sao, sao ? nCtu : 0);
  st.add(&A.alf.ctus, p->alf, alf ? nCtu : 0); stage_alf_tables(st, A.alf, alf ? p->alfTabs : nullptr);
  st.add(&A.mc.dmvrMv, nullptr, p->numDmvr * 2);
  st.add(&A.mc.wp, p->wp, p->numWp);
  st.add(&A.lm.lmcs, p->lmcs, lm ? 1 : 0); st.add(&A.lm.invLut, lm ? p->lmcs->invLUT : nullptr, lm ? 1 << g.bitDepth : 0);
  st.add(&A.lm.vpdus, lm && p->lmcs->chromaAdj ? p->lmcs->vpdus : nullptr, lm ? nVpdu : 0); st.add(&A.lm.scale, nullptr, lm ? nVpdu : 0);
  stage_picture(st, A.given, given ? p->given : nullptr, g, given);
  st.add(&A.intra.tus, p->intraTus, ni); st.add(&A.intra.sync, nullptr, ni ? ni + 2 : 0); st.add(&A.intra.order, nullptr, ni ? intra_order_ints(g, ni) : 0);
  for (int k = 0; k < (g.chromaFormat ? 3 : 1) && ni; k++) st.add(&A.intra.owner[k], nullptr, A.intra.ownerBytes[k] / sizeof(int));
  if (ni) if (int rc = c->resiBuf.reserve(c->picBytes)) return rc;
  if (st.bytes() > A.buf.cap) { B200_CUDA(cudaStreamSynchronize(c->stream)); B200_CUDA(cudaStreamSynchronize(c->upStream)); A.donePending = false; }   // realloc: nothing may still use the old buffer
  cudaStream_t s = c->upStream;                                       // H2D on its own stream: overlaps the kernels of earlier pictures
  if (A.donePending) { B200_CUDA(cudaStreamWaitEvent(s, A.done, 0)); A.donePending = false; }   // kernels of the arena's previous picture
  if (int rc = st.commit(A.buf, s)) return rc;
  if (!lf || !p->ctuSlice) A.lf.ctuSlice = nullptr;                   // the entry is there either way, uploaded only for deblocking
  if (p->numDmvr) B200_CUDA(cudaMemsetAsync(A.mc.dmvrMv, 0, p->numDmvr * 8, s));   // entries of non-DMVR CUs stay zero, like m_dmvrMvCache users expect
  if (lf) lf_tables(A.lf, p->lfSlices, p->numLfSlices, p->lfSeq);
  A.lfd.numCus = lfd ? p->numLfCus : 0;
  if (lfd) {
    A.lfd.anyDisabled = false;
    for (int k = 0; k < p->numLfSlices; k++) A.lfd.anyDisabled = A.lfd.anyDisabled || p->lfSlices[k].disable;
    A.lfd.geom = g; A.lfd.map[1] = A.lfd.map[0] + n4; A.lfd.pus = A.mc.pus; A.lfd.numPus = p->numPus; A.lfd.lfV = const_cast<b200_lf_param*>(A.lf.lfV); A.lfd.lfH = const_cast<b200_lf_param*>(A.lf.lfH);
  }
  A.lf.dirs = 3;
  if (sao) { if (p->vb) A.sao.vb = *p->vb; else memset(&A.sao.vb, 0, sizeof(A.sao.vb)); }
  for (int k = 0; k < 3; k++) A.mc.refStride[k] = g.stride[k];
  A.mc.lmcs = A.lm.lmcs; A.lmcsChromaAdj = lm && p->lmcs->chromaAdj;
  A.mc.tiles = tiles; A.mc.meta = meta; A.k1.idx = tuIdx; A.k1.meta = meta + LM_INTS;
  A.numPus = p->numPus; A.numDmvr = p->numDmvr; A.k1.numTus = p->numTus; A.k1.mode = 0; A.intra.numTus = ni;
  const DevPlanes resi = ni ? pic_planes(c->resiBuf.p, g) : DevPlanes();
  for (int k = 0; k < 3; k++) { A.k1.resi[k] = resi.p[k]; A.intra.resi[k] = resi.p[k]; }
  A.ciipResi = false;
  for (size_t i = 0; i < ni && !A.ciipResi; i++) { const b200_intra_tu& t = p->intraTus[i]; A.ciipResi = t.ciip && !(t.flags & B200_INTRA_ISP) && (t.flags & B200_INTRA_ADD_RESI); }
  A.dstSlot = p->dstSlot; A.flags = p->flags; A.valid = true;
  // work lists: validated and bucketed on the device, behind the copies
  KHook* h = &c->hook;
  if (int rc = launch_mc_bucket(A.mc.pus, p->numPus, tiles, capTiles, meta, g, c->numSlots, p->numWp, p->numDmvr, s, h)) return rc;
  if (int rc = launch_tu_bucket(A.k1.tus, p->numTus, tuIdx, meta + LM_INTS, g, p->numCoefs, p->numScaling, s, h)) return rc;
  if (int rc = launch_ctu_validate(A.sao.ctus, A.alf.ctus, A.lf.ctuSlice, (int)nCtu, ctu_limits(g, alf ? p->alfTabs : nullptr, p->numLfSlices), meta, s, h)) return rc;
  if (int rc = launch_intra_validate(A.intra.tus, ni, g, meta, s, h)) return rc;
  if (A.lmcsChromaAdj) if (int rc = launch_lmcs_validate(A.lm.vpdus, g, meta, s, h)) return rc;
  if (lfd) if (int rc = launch_lf_validate(A.lfd.cus, p->numLfCus, A.lfd.tus, p->numLfTus, A.lfd.ctuCus, g, p->numLfSlices, meta, s, h)) return rc;
  B200_CUDA(cudaMemcpyAsync(A.hMeta, meta, 2 * LM_INTS * sizeof(int), cudaMemcpyDeviceToHost, s));   // list lengths for b200_pic_run's grids
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
  B200_CHECK(!(A.hMeta[LM_ERR] & LM_ERR_LF_RECORD), "b200_pic_run: a CU / TU record of the edge derivation is invalid (block outside its plane or CTU, slice or TU index out of range, CTU ranges)");
  B200_CHECK(!A.hMeta[LM_INTS + LM_ERR], "b200_pic_run: the picture's TU list holds an invalid record");
  B200_CUDA(cudaStreamWaitEvent(s, A.uploaded, 0));
  const b200_geom& g = c->g;
  KHook* h = &c->hook;
  int cur = c->work[0], other = c->work[1];
  for (int b : {cur, other}) if (int rc = wait_readers(c, b)) return rc;   // async outputs still reading these buffers
  DevPlanes P = c->planes(cur);
  // 0. pre-reconstructed (intra stand-in) samples
  if (A.given.p[0]) {
    for (int k = 0; k < (g.chromaFormat ? 3 : 1); k++) B200_CUDA(cudaMemcpyAsync(P.p[k], A.given.p[k], plane_bytes(g, k), cudaMemcpyDeviceToDevice, s));
  }
  // 1. K2 inter prediction
  if (A.numPus) {
    A.mc.dst = P;
    for (int sl = 0; sl < c->numSlots; sl++) { DevPlanes d = c->planes(c->slotBuf[sl]); for (int k = 0; k < 3; k++) A.mc.refs[sl * 3 + k] = d.p[k]; }
    for (int l = 0; l < MC_LISTS; l++) A.mc.cnt[l] = A.hMeta[LM_CNT + l];
    if (int rc = launch_mc(A.mc, c->ss, h)) return rc;
  }
  // 2. K1 residual + reco, 2b. K6 intra blocks in decoding order (prediction from the reconstruction so far — inter CUs, earlier intra blocks — + their
  // residual).  With LMCS chroma scaling the chroma residual scale of a VPDU is derived from its reconstructed (mapped-domain) luma neighbourhood
  // (Reshape.cpp:192), intra blocks included: luma TUs -> luma intra blocks -> per-VPDU scale -> chroma TUs (scaled) -> chroma intra blocks.
  A.k1.planes = A.intra.planes = A.lm.planes = P;
  for (int l = 0; l < K1_LISTS; l++) A.k1.cnt[l] = A.hMeta[LM_INTS + LM_CNT + l];
  const bool twoPass = A.lm.lmcs && A.lmcsChromaAdj;
  A.hMeta[2 * LM_INTS] = 0;
  if (A.ciipResi) if (int rc = launch_intra_ciip_clear(A.intra.tus, A.intra.numTus, A.k1.resi, P.stride, s, h)) return rc;
  auto runK1 = [&](int compSel, const int* vpduScale) -> int {
    if (!A.k1.numTus) return 0;
    A.k1.compSel = compSel; A.k1.vpduScale = vpduScale;
    return launch_k1_residual(A.k1, c->ss, h);
  };
  auto runK6 = [&](int compSel) -> int { A.intra.compSel = compSel; return launch_intra(A.intra, s, h); };
  if (twoPass) {
    if (int rc = runK1(1, nullptr)) return rc;
    if (int rc = runK6(1)) return rc;
    if (int rc = launch_lmcs_vpdu(A.lm, s, h)) return rc;
    if (int rc = runK1(2, A.lm.scale)) return rc;
    if (int rc = runK6(2)) return rc;
  } else {
    if (int rc = runK1(0, nullptr)) return rc;
    if (int rc = runK6(0)) return rc;
  }
  if (A.intra.numTus) B200_CUDA(cudaMemcpyAsync(A.hMeta + 2 * LM_INTS, A.intra.sync + A.intra.numTus + 1, sizeof(int), cudaMemcpyDeviceToHost, s));   // timeout bit, read by b200_wait_picture
  if (A.lm.lmcs) if (int rc = launch_lmcs_inv(A.lm, s, h)) return rc;   // RSP stage (DecLibRecon.cpp:935)
  // 3. K3 deblocking
  if (A.flags & B200_PIC_DEBLOCK) {
    A.lf.planes = P;
    if (A.lfd.numCus) if (int rc = launch_lf_derive(A.lfd, s, h)) return rc;
    if (int rc = launch_lf_deblock(A.lf, s, h)) return rc;
  }
  // 4. K4 SAO (out of place)
  if (A.flags & B200_PIC_SAO) {
    A.sao.src = P; A.sao.dst = c->planes(other);
    if (int rc = launch_sao(A.sao, s, h)) return rc;
    std::swap(cur, other); P = c->planes(cur);
  }
  // 5. K5 ALF (out of place, straight into a buffer that becomes the DPB slot)
  if (A.flags & B200_PIC_ALF) {
    A.alf.src = P; A.alf.dst = c->planes(other);
    if (int rc = launch_alf(A.alf, c->ss, h)) return rc;
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
  if (dmvrMv && ai >= 0 && ai < c->numArenas && c->arenas[ai].mc.dmvrMv) {
    const size_t n = numDmvr < c->arenas[ai].numDmvr ? numDmvr : c->arenas[ai].numDmvr;
    if (n) { if (int rc = copy_host(dmvrMv, c->arenas[ai].mc.dmvrMv, n * 8, cudaMemcpyDeviceToHost, c->stream)) return rc; }
  }
  B200_CUDA(cudaStreamSynchronize(c->upStream));
  B200_CUDA(cudaStreamSynchronize(c->stream));
  if (ai >= 0 && ai < c->numArenas && c->arenas[ai].intra.numTus) {
    const int err = c->arenas[ai].hMeta[2 * LM_INTS];
    B200_CHECK(!(err & INTRA_ERR_CTU_BLOCKS), "b200_wait_picture: a CTU holds more than %d intra block records (overlapping records?)", INTRA_MAX_CTU_BLOCKS);
    B200_CHECK(!err, "b200_wait_picture: an intra block waited for a neighbour that never finished (intra list not in decoding order?)");
  }
  return 0;
}

B200_API int b200_get_frame(b200_ctx* c, int slot, int16_t* const planes[3])
{
  B200_CHECK(c && planes && slot >= 0 && slot < c->numSlots, "b200_get_frame: bad argument");
  return copy_slot(c, slot, planes, nullptr, cudaMemcpyDeviceToHost, "b200_get_frame");
}

B200_API int b200_ctx_load_slot_strided(b200_ctx* c, int slot, const int16_t* const planes[3], const ptrdiff_t strides[3])
{
  B200_CHECK(c && planes && strides && slot >= 0 && slot < c->numSlots, "b200_ctx_load_slot_strided: bad argument");
  return copy_slot(c, slot, const_cast<int16_t* const*>(planes), strides, cudaMemcpyHostToDevice, "b200_ctx_load_slot_strided");
}

B200_API int b200_get_frame_strided(b200_ctx* c, int slot, int16_t* const planes[3], const ptrdiff_t strides[3])
{
  B200_CHECK(c && planes && strides && slot >= 0 && slot < c->numSlots, "b200_get_frame_strided: bad argument");
  return copy_slot(c, slot, planes, strides, cudaMemcpyDeviceToHost, "b200_get_frame_strided");
}

// An asynchronous read of a slot's buffer on stream s starts after everything submitted so far (this slot's picture included) and ends with mark_read;
// a read that returns a ticket takes it after its last copy.
static int begin_read(b200_ctx* c, int slot, cudaStream_t s, DevPlanes* d)
{
  B200_CUDA(cudaEventRecord(c->finalEv, c->stream));
  B200_CUDA(cudaStreamWaitEvent(s, c->finalEv, 0));
  *d = c->planes(c->slotBuf[slot]);
  return 0;
}

static int take_ticket(b200_ctx* c, cudaStream_t s)
{
  const int t = c->nextTicket; c->nextTicket = (c->nextTicket + 1) & 15;
  B200_CUDA(cudaEventRecord(c->ticketEv[t], s));
  return t;
}

// whole planes of d (strides, padding included) to the caller's planes, on the copy stream
static int download_planes(b200_ctx* c, const DevPlanes& d, void* const planes[3])
{
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++) if (int rc = copy_host(planes[k], d.p[k], plane_bytes(c->g, k), cudaMemcpyDeviceToHost, c->copyStream)) return rc;
  return 0;
}

// Output stage st for a frame in fmt (pyuv / 8 bit): plane k at dst[k], bytes[k] long.  Reserved before the copy stream is ordered after the kernels, so
// that growing it waits only for earlier copies.
static int out_stage(b200_ctx* c, int fmt, int st, uint8_t* dst[3], size_t bytes[3])
{
  size_t off[3] = {0, 0, 0}, total = 0;
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++) { bytes[k] = b200_frame_bytes(&c->g, fmt, k); off[k] = total; total += align256(bytes[k]); }
  if (total > c->outStage[st].cap) B200_CUDA(cudaStreamSynchronize(c->copyStream));          // growing: no copy may still read the old block
  if (int rc = c->outStage[st].reserve(total)) return rc;
  for (int k = 0; k < 3; k++) dst[k] = c->outStage[st].as<uint8_t>() + off[k];
  return 0;
}

// d converted to fmt in the output stage dst and downloaded to the caller's planes, on the copy stream; when d is a slot's buffer (slot >= 0) the
// buffer is free once it is packed
static int pack_download(b200_ctx* c, const DevPlanes& d, int fmt, uint8_t* const dst[3], const size_t bytes[3], void* const planes[3], int slot)
{
  if (int rc = launch_pack(d, c->g, fmt, dst, c->copyStream, &c->hook)) return rc;           // on the copy stream: the kernel stream runs on
  if (slot >= 0) if (int rc = mark_read(c, c->slotBuf[slot], c->copyStream)) return rc;
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++) if (int rc = copy_host(planes[k], dst[k], bytes[k], cudaMemcpyDeviceToHost, c->copyStream)) return rc;
  return 0;
}

B200_API int b200_get_frame_async(b200_ctx* c, int slot, int16_t* const planes[3])
{
  B200_CHECK(c && planes && slot >= 0 && slot < c->numSlots, "b200_get_frame_async: bad argument");
  DevPlanes d;
  if (int rc = begin_read(c, slot, c->copyStream, &d)) return rc;
  void* const out[3] = {planes[0], planes[1], planes[2]};
  if (int rc = download_planes(c, d, out)) return rc;
  if (int rc = mark_read(c, c->slotBuf[slot], c->copyStream)) return rc;
  return take_ticket(c, c->copyStream);
}

// Device-to-device output on a stream of the caller's (multi-GPU gather: the frame goes to a send buffer, NCCL takes it from there): the caller's stream
// waits for everything submitted so far, the copies run on it, and later pictures wait for them before they overwrite the DPB buffer.
B200_API int b200_get_frame_device_async(b200_ctx* c, int slot, int16_t* const planesDev[3], void* cudaStream)
{
  B200_CHECK(c && planesDev && slot >= 0 && slot < c->numSlots, "b200_get_frame_device_async: bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(cudaStream);
  DevPlanes d;
  if (int rc = begin_read(c, slot, st, &d)) return rc;
  for (int k = 0; k < (c->g.chromaFormat ? 3 : 1); k++) {
    B200_CHECK(planesDev[k], "b200_get_frame_device_async: plane %d", k);
    B200_CUDA(cudaMemcpyAsync(planesDev[k], d.p[k], plane_bytes(c->g, k), cudaMemcpyDeviceToDevice, st));
  }
  return mark_read(c, c->slotBuf[slot], st);
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
  const int st = c->nextStage; c->nextStage ^= 1;
  uint8_t* dst[3]; size_t bytes[3] = {0, 0, 0};
  if (int rc = out_stage(c, fmt, st, dst, bytes)) return rc;
  DevPlanes d;
  if (int rc = begin_read(c, slot, c->copyStream, &d)) return rc;
  if (int rc = pack_download(c, d, fmt, dst, bytes, planes, slot)) return rc;
  return take_ticket(c, c->copyStream);
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
  const int nbx = (g.width + 15) / 16, nby = (g.height + 15) / 16;
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
  DevPlanes src;
  if (int rc = begin_read(c, slot, c->copyStream, &src)) return rc;
  const DevPlanes gr = pic_planes(c->grainStage[st].p, g);
  if (int rc = launch_film_grain(src, gr, g, reinterpret_cast<const int8_t*>(tb), tb + oS, tb + oP, reinterpret_cast<const uint32_t*>(tb + oL),
                                 reinterpret_cast<uint32_t*>(tb + oB), fg->scaleShift, fg->compPresent, c->copyStream, &c->hook)) return rc;
  if (int rc = mark_read(c, c->slotBuf[slot], c->copyStream)) return rc;                      // the picture buffer is free once the grained copy exists
  if (fmt == B200_OUT_16) { if (int rc = download_planes(c, gr, planes)) return rc; }
  else {
    uint8_t* dst[3]; size_t bytes[3] = {0, 0, 0};
    if (int rc = out_stage(c, fmt, st, dst, bytes)) return rc;
    if (int rc = pack_download(c, gr, fmt, dst, bytes, planes, -1)) return rc;
  }
  return take_ticket(c, c->copyStream);
}

B200_API int b200_frame_hash_async(b200_ctx* c, int slot, int method, uint8_t* digest)
{
  B200_CHECK(c && digest && slot >= 0 && slot < c->numSlots, "b200_frame_hash_async: bad argument");
  if (method == B200_HASH_MD5) { set_error("b200_frame_hash_async: MD5 is a serial chain over each plane and is not computed on the device; use CRC or checksum"); return B200_ERR_UNSUPPORTED; }
  B200_CHECK(method == B200_HASH_CRC || method == B200_HASH_CHECKSUM, "b200_frame_hash_async: unknown method %d", method);
  B200_CUDA(cudaSetDevice(c->device));
  if (int rc = c->hashBuf.reserve(16 * 32)) return rc;                                        // per ticket: 3 accumulators + 12 digest bytes
  uint32_t* acc = c->hashBuf.as<uint32_t>() + c->nextTicket * 8; uint8_t* dig = reinterpret_cast<uint8_t*>(acc + 4);   // the slot of the ticket this call takes
  DevPlanes d;
  if (int rc = begin_read(c, slot, c->copyStream, &d)) return rc;
  B200_CUDA(cudaMemsetAsync(acc, 0, 32, c->copyStream));
  if (int rc = launch_hash(d, c->g, method, acc, dig, c->copyStream, &c->hook)) return rc;
  if (int rc = mark_read(c, c->slotBuf[slot], c->copyStream)) return rc;
  if (int rc = copy_host(digest, dig, 12, cudaMemcpyDeviceToHost, c->copyStream)) return rc;
  return take_ticket(c, c->copyStream);
}

B200_API int b200_frame_wait(b200_ctx* c, int ticket)
{
  B200_CHECK(c && ticket >= 0 && ticket < 16, "b200_frame_wait: bad ticket");
  B200_CUDA(cudaEventSynchronize(c->ticketEv[ticket]));
  return 0;
}

B200_API int b200_ctx_mark(b200_ctx* c, int which) { B200_CHECK(c && (which == 0 || which == 1), "b200_ctx_mark"); B200_CUDA(cudaEventRecord(c->ev[which], c->stream)); return 0; }
B200_API int b200_ctx_elapsed_ms(b200_ctx* c, float* ms) { B200_CHECK(c && ms, "b200_ctx_elapsed_ms"); B200_CUDA(cudaEventSynchronize(c->ev[1])); B200_CUDA(cudaEventElapsedTime(ms, c->ev[0], c->ev[1])); return 0; }
B200_API long long b200_ctx_kernel_launches(b200_ctx* c) { return c ? c->hook.launches : 0; }

B200_API int b200_ctx_set_profiling(b200_ctx* c, int on) { B200_CHECK(c, "b200_ctx_set_profiling"); c->hook.profiling = on != 0; return 0; }

B200_API int b200_ctx_get_kernel_ms_n(b200_ctx* c, float* ms, int* counts, int n)
{
  B200_CHECK(c && ms && counts && n >= 1 && n <= B200_KF_COUNT, "b200_ctx_get_kernel_ms_n");
  B200_CUDA(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < n; i++) { ms[i] = 0; counts[i] = 0; }
  for (auto& r : c->hook.recs) { float t = 0; cudaEventElapsedTime(&t, r.a, r.b); if (r.family < n) { ms[r.family] += t; counts[r.family]++; } c->hook.pool.push_back(r.a); c->hook.pool.push_back(r.b); }
  c->hook.recs.clear();
  return 0;
}
B200_API int b200_ctx_get_kernel_ms(b200_ctx* c, float ms[8], int counts[8]) { return b200_ctx_get_kernel_ms_n(c, ms, counts, 8); }

B200_API int b200_host_register(void* ptr, size_t bytes) { B200_CHECK(ptr && bytes, "b200_host_register"); if (int rc = ensure_device()) return rc; B200_CUDA(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault)); return 0; }
B200_API int b200_host_unregister(void* ptr) { B200_CHECK(ptr, "b200_host_unregister"); B200_CUDA(cudaHostUnregister(ptr)); return 0; }

}  // extern "C"
