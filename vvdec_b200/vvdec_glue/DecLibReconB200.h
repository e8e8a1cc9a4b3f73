// DecLibReconB200.h — the drop-in for DecLibRecon (reference DecoderLib/DecLibRecon.h:143-200): the same methods with the same signatures
// and the same contract — create( ThreadPool*, unsigned, bool ), destroy(), decompressPicture( Picture* ), waitForPrevDecompressedPic(),
// cleanupOnException(), getCurrPic() — reconstruction on the GPU through the C ABI of include/vvdec_b200.h.  Header-only glue that lives INSIDE a
// VVdeC build (INTEGRATION.md).  It is compiled against the reference headers by oracle/Makefile.ref and EXECUTED by oracle/ref_seam.h: the stock
// DecLibRecon and this class reconstruct the same parsed Picture, bit-exactly (tests/test_seam_*.py).  Its building blocks — flattenTU, flattenPU /
// flattenSbTmvp, flattenIntraTU / flattenCiipBlock, flattenSAO / flattenALF / buildAlfTables / flattenLfCtu — are also pinned one by one.
//
// decompressPicture() returns at once, like the reference's (DecLibRecon.cpp:429-681): the host stages run as tasks of the decoder's thread pool,
//   MIDER   one task per CTU row, wave front over rows (DecCu::TaskDeriveCtuMotionInfo, the MIDER case of ctuTask :762-781): the task walks its CTUs as far
//           as the row above allows and hands itself back to the pool when it has to wait; may start while the rows below are still being parsed
//           (ctuParsedBarrier, RECO_WHILE_PARSE)
//   FLATTEN one task per run of three CTUs, ready when their motion is derived: boundary strengths (calcFilterStrengthsCTU, the LF_INIT case :808-829),
//           the CU / TU walk of TaskTrafoCtu / TaskInterCtu / TaskCriticalIntraKernel (DecCu.cpp:106-159) into per-CTU work lists
//   SUBMIT  one task: lists joined in CTU order (K6 needs decoding order), SAO / ALF CTU records, per-slice tables, b200_decompress_picture (stream-ordered
//           behind the pictures it references, also those another recon instance is still flattening)
// and waitForPrevDecompressedPic() waits for the device, takes the DMVR deltas, runs TaskFinishMotionInfo (DecCu.cpp:161) and copies the
// finished planes into Picture::m_bufs (output / CPU fallback of later pictures).
// Errors follow DecLibRecon.cpp:684-722: the first exception of a picture is parked (no task lets one escape into the pool), waitForPrevDecompressedPic()
// rethrows it, sets pic->error and reconDone.setException() and clears the pool of this picture's tasks (cleanupOnException).  B200_ERR_UNSUPPORTED maps to
// UnsupportedFeatureException, B200_ERR_PARAM to RecoverableException, every other failure to Exception (TypeDef.h:828-831).
//
// The CPU keeps: parsing, motion derivation, boundary strengths, TaskFinishMotionInfo.  Pictures that use a tool the device path does not
// have throw UnsupportedFeatureException (see refuse() below for the list); a deployment keeps a stock DecLibRecon next to this class and
// routes those pictures to it — their output is imported into the device DPB when a later picture references it (importReference).
// DecLib owns two recon instances that alternate (DecLib.h:70): the device context and its DPB bookkeeping are shared by all instances
// created with the same ThreadPool.
#pragma once
#include <vector>
#include <map>
#include <mutex>
#include <memory>
#include <atomic>
#include <chrono>
#include "vvdec_b200.h"
#include "flatten_tu.h"
#include "flatten_pu.h"
#include "flatten_filters.h"
#include "flatten_intra.h"
#include "../csrc/vvc_tables.h"
#include "../csrc/lf_derive.cuh"
#include "CommonLib/Picture.h"
#include "CommonLib/LoopFilter.h"
#include "CommonLib/Reshape.h"
#include "CommonLib/Quant.h"
#include "CommonLib/WeightPrediction.h"
#include "CommonLib/InterPrediction.h"
#include "DecoderLib/DecCu.h"
#include "Utilities/ThreadPool.h"

namespace b200glue
{
using namespace vvdec;

// grow-only pinned host array (cudaHostRegister through the C ABI: the memory stays owned by the vector)
template<class T> struct PinnedVec
{
  std::vector<T> v; const void* reg = nullptr; size_t regBytes = 0;
  void clear() { v.clear(); }
  void pin() { if( v.capacity() * sizeof( T ) != regBytes || (const void*) v.data() != reg ) { if( reg ) b200_host_unregister( const_cast<void*>( reg ) ); reg = nullptr; regBytes = 0; if( v.capacity() && b200_host_register( v.data(), v.capacity() * sizeof( T ) ) == 0 ) { reg = v.data(); regBytes = v.capacity() * sizeof( T ); } } }
  ~PinnedVec() { if( reg ) b200_host_unregister( const_cast<void*>( reg ) ); }
};

class DecLibReconB200
{
  // ---- device context + DPB bookkeeping, shared by the recon instances of one decoder ----
  struct Shared
  {
    std::mutex m; b200_ctx* ctx = nullptr; b200_geom geom{}; int numSlots = 0;
    // valid[slot]: 0 nothing usable; 1 the owner's final samples are resident; 2 the owner is being reconstructed by a recon instance and its work is not yet
    // in the stream; 3 ... and has been submitted (whatever is submitted later reads the finished samples: one stream, in order)
    std::map<const Picture*, int> slotOf; std::vector<const Picture*> owner; std::vector<uint8_t> valid;
    std::vector<DecLibReconB200*> instances;                                   // the recon instances on this pool (DecLib keeps two, DecLib.h:70)
    ~Shared() { if( ctx ) b200_ctx_destroy( ctx ); }
  };
  static std::shared_ptr<Shared> sharedFor( const void* key )
  {
    static std::mutex m; static std::map<const void*, std::weak_ptr<Shared>> reg;
    std::lock_guard<std::mutex> l( m );
    std::shared_ptr<Shared> s = reg[key].lock();
    if( !s ) { s = std::make_shared<Shared>(); reg[key] = s; }
    return s;
  }
  std::shared_ptr<Shared> m_sh;

  // ---- per-CTU work lists (one pool task per CTU: MIDER, then boundary strengths + flatten of the same CTU) ----
  struct Row
  {
    DecLibReconB200* self = nullptr; int line = 0, col = 0;
    std::vector<b200_pu> pus; std::vector<b200_tu> tus; std::vector<int16_t> coefs; std::vector<b200_intra_tu> intra;
    std::vector<b200_lf_cu> lfCus; std::vector<b200_lf_tu> lfTus;       // setDeviceLfDerive: the records the device derives the edge grids from
  };

  ThreadPool* m_pool = nullptr; int m_numThreads = 1; unsigned m_id = 0; int m_dpbSlots = 17;
  std::atomic<long long> m_cpuNs[5] = {};   // CPU time of the host stages summed over the pool's threads: MIDER, Bs + grid copy, CU / TU walk, submit, finish
  struct CpuTimer { std::atomic<long long>& acc; std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now(); ~CpuTimer() { acc += std::chrono::duration_cast<std::chrono::nanoseconds>( std::chrono::steady_clock::now() - t0 ).count(); } };
  std::vector<int> m_waitSlots;            // slots of reference pictures that were in flight on another instance when this picture was set up
  Picture*    m_currDecompPic = nullptr;
  int         m_arena = -1, m_dstSlot = -1;
  std::vector<Row> m_rows; int m_ctusW = 0;
  std::vector<MotionHist> m_hist;
  WaitCounter m_flattenCounter, m_submitCounter, m_finishCounter, m_doneCounter;
  std::recursive_mutex m_finishMutex; bool m_asyncFinish = false; std::vector<int> m_refSlots;
  // per-picture work lists (pinned)
  PinnedVec<b200_pu> m_pus; PinnedVec<b200_tu> m_tus; PinnedVec<int16_t> m_coefs; PinnedVec<b200_intra_tu> m_intra;
  PinnedVec<b200_lf_param> m_lf[2]; PinnedVec<b200_sao_ctu> m_sao; PinnedVec<b200_alf_ctu> m_alf; PinnedVec<b200_lmcs_vpdu> m_vpdus;
  PinnedVec<int32_t> m_dmvr;
  PinnedVec<b200_lf_cu> m_lfCus; PinnedVec<b200_lf_tu> m_lfTus; PinnedVec<uint32_t> m_lfCtuCus; std::vector<uint8_t> m_lfSliceB;
  bool m_lfDerive = false, m_lfOn = false;  // setDeviceLfDerive; whether the current picture uses it
  std::vector<b200_wp> m_wp; int m_wpStride = 0; std::vector<int> m_wpIdx;
  AlfTableStore m_alfStore; b200_alf_tables m_alfTabs{}; b200_lmcs m_lmcs{}; b200_vb m_vb{}; b200_lf_slice m_lfSlice{}; b200_lf_seq m_lfSeq{};
  b200_picture m_pic{};
  SlotMap m_slotMap{};
  // per slice of the picture (pic->slices order): reference slots, weighted-prediction index table, bases of its ALF sets in the picture-level tables
  struct SliceTabs { const Slice* slice = nullptr; SlotMap slotMap{}; std::vector<int> wpIdx; int wpStride = 0; AlfSliceBase alf; };
  std::vector<SliceTabs> m_sl; std::vector<b200_lf_slice> m_lfSlices; PinnedVec<uint8_t> m_ctuSlice;
  int sliceIdx( const Slice* s ) const { for( size_t i = 0; i < m_sl.size(); i++ ) if( m_sl[i].slice == s ) return (int) i; THROW_FATAL( "DecLibReconB200: a CU of a slice the picture does not list" ); }
  bool m_doSao = false, m_doAlf = false, m_doLmcs = false, m_dryRun = false;
  bool m_finished = false;                 // the current picture has been finished ahead of waitForPrevDecompressedPic() (finishCollocatedPictures)
  // host-stage timing (seconds since decompressPicture): end of preparePicture, first flatten row start (= MIDER done), submit start, submit end, wait end
  std::chrono::steady_clock::time_point m_t0; std::atomic<int64_t> m_tFlat0{ 0 }; double m_stage[6] = { 0, 0, 0, 0, 0, 0 };
  double since() const { return std::chrono::duration<double>( std::chrono::steady_clock::now() - m_t0 ).count(); }
  // the CPU stages that stay
  std::vector<MotionInfo> m_motionInfo; std::vector<LoopFilterParam> m_loopFilterParam; std::vector<Mv> m_dmvrMvCache;
  // explicit scaling lists: the reference's own table set (Quant::init -> setScalingListDec, Quant.cpp:386) in one contiguous buffer; a TU's table is addressed by its
  // offset in it (b200_tu::slOff).  TrQuant derives privately from Quant, so the glue keeps a Quant of its own for the tables
  std::unique_ptr<Quant> m_quant; bool m_useSL = false; const int* m_slBase = nullptr; size_t m_slCount = 0; const void* m_slReg = nullptr;
  // Pinned pages that stay registered after their memory is freed keep the old physical pages: a later allocation at the same address would then be copied
  // from / to those pages instead of its own.  The scaling tables are unregistered before they move or go away.
  void unpinScaling() { if( m_slReg ) b200_host_unregister( const_cast<void*>( m_slReg ) ); m_slReg = nullptr; }
  void setSlOff( const CodingUnit& cu, b200_tu& t ) const
  {
    if( !( t.flags & B200_TU_SCALING ) ) return;
    const int list = ( CU::isIntra( cu ) ? 0 : MAX_NUM_COMPONENT ) + t.comp;                  // getScalingListType, Quant.cpp:289
    t.slOff = (uint32_t) ( m_quant->getDequantCoeff( list, t.log2w, t.log2h ) - m_slBase );
  }
  struct AlfAccess : AdaptiveLoopFilter { using AdaptiveLoopFilter::isClipOrCrossedByVirtualBoundaries; };     // protected in the reference: the glue asks it per CTU
  LoopFilter m_cLoopFilter; SampleAdaptiveOffset m_cSAO; AlfAccess m_cALF; Reshape m_cReshaper;
  std::vector<std::unique_ptr<DecCu>> m_cuDecoders; InterPrediction m_interPred; std::unique_ptr<TrQuant> m_trQuant;
  PelStorage m_fltBuf; ChromaFormat m_fltFmt = CHROMA_420; int m_fltCtu = 0;

  static void check( int rc ) { if( rc == B200_ERR_UNSUPPORTED ) THROW_UNSUPPORTED( b200_last_error() ); if( rc == B200_ERR_PARAM ) THROW_RECOVERABLE( b200_last_error() ); if( rc < 0 ) THROW_FATAL( b200_last_error() ); }

  // ---- DPB slots.  A picture the device did not reconstruct itself (CPU fallback, lost picture filled grey) is uploaded when it is first referenced.
  int slotLocked( const Picture* pic )
  {
    Shared& S = *m_sh;
    auto it = S.slotOf.find( pic ); if( it != S.slotOf.end() ) return it->second;
    for( int s = 0; s < S.numSlots; s++ )
      if( !S.owner[s] || ( !S.owner[s]->stillReferenced && S.owner[s]->progress >= Picture::reconstructed && S.owner[s] != m_currDecompPic ) )
      { if( S.owner[s] ) S.slotOf.erase( S.owner[s] ); S.owner[s] = pic; S.valid[s] = 0; S.slotOf[pic] = s; return s; }
    THROW_FATAL( "DecLibReconB200: device DPB is full" );
  }
  int importReference( const Picture* ref )
  {
    Shared& S = *m_sh;
    const int s = slotLocked( ref );
    if( S.valid[s] == 1 || S.valid[s] == 3 ) return s;
    if( S.valid[s] == 2 ) { m_waitSlots.push_back( s ); return s; }        // the other recon instance has it in flight: this picture is submitted behind it (submitReady)
    CHECK_FATAL( ref->progress < Picture::reconstructed, "DecLibReconB200: reference picture is neither on the device nor reconstructed on the host" );
    const int16_t* planes[3] = { nullptr, nullptr, nullptr }; ptrdiff_t strides[3] = { 0, 0, 0 };
    for( int c = 0; c < ( S.geom.chromaFormat ? 3 : 1 ); c++ ) { const CPelBuf b = ref->getRecoBuf( ComponentID( c ) ); planes[c] = b.buf; strides[c] = b.stride; }
    if( (int) ref->getRecoBuf( COMPONENT_Y ).width != S.geom.width || (int) ref->getRecoBuf( COMPONENT_Y ).height != S.geom.height ) THROW_UNSUPPORTED( "DecLibReconB200: reference picture of another size (RPR)" );
    if( !m_dryRun ) check( b200_ctx_load_slot_strided( S.ctx, s, planes, strides ) );
#ifdef B200_GLUE_TEST_HOOKS
    else if( testHooks().loadSlot ) testHooks().loadSlot( testHooks().user, s, planes, strides, &S.geom );
#endif
    S.valid[s] = 1;
    return s;
  }

  // ---- what the device path does not have: the picture goes to the stock DecLibRecon ----
  void refuse( const Picture* pic ) const
  {
    const CodingStructure& cs = *pic->cs; const SPS& sps = *cs.sps; const PPS& pps = *cs.pps;
    if( sps.getChromaFormatIdc() != CHROMA_420 && sps.getChromaFormatIdc() != CHROMA_400 ) THROW_UNSUPPORTED( "DecLibReconB200: 4:2:0 and 4:0:0 only" );
    if( sps.getUseWrapAround() || pic->subPictures.size() > 1 || cs.picHeader->getVirtualBoundariesPresentFlag() ) THROW_UNSUPPORTED( "DecLibReconB200: wrap-around / sub-pictures / virtual boundaries" );
    if( pic->slices.size() > 64 ) THROW_UNSUPPORTED( "DecLibReconB200: more than 64 slices in a picture" );
    for( const Slice* sl : pic->slices )
    {
      if( sl->getLmcsEnabledFlag() != pic->slices[0]->getLmcsEnabledFlag() ) THROW_UNSUPPORTED( "DecLibReconB200: LMCS switched per slice" );
    }
    // A CIIP CU larger than the maximum transform size codes every luma cbf and may end up without any coefficient; the parser then clears rootCbf
    // (CABACReader.cpp:1449-1456) and the reference maps the blended block through the LMCS forward curve a SECOND time (DecCu.cpp:466-476, the `else` branch runs in
    // the inter pass and again in the CIIP pass).  Only possible with sps_max_luma_transform_size_64_flag == 0; the device path (one forward map, as the standard
    // has it) would differ from the reference there, so those pictures are left to the stock back end.
    if( sps.getLog2MaxTbSize() < 6 && sps.getCTUSize() > ( 1u << sps.getLog2MaxTbSize() ) && sps.getUseCiip() && pic->slices[0]->getLmcsEnabledFlag() && std::any_of( pic->slices.begin(), pic->slices.end(), []( const Slice* sl ) { return !sl->isIntra(); } ) )
      THROW_UNSUPPORTED( "DecLibReconB200: CIIP under LMCS with 32x32 maximum transform size (the reference's double forward mapping of residual-free CIIP blocks)" );
    if( sps.getIBCFlag() ) THROW_UNSUPPORTED( "DecLibReconB200: IBC" );
    if( sps.getUseColorTrans() ) THROW_UNSUPPORTED( "DecLibReconB200: adaptive colour transform" );
  }

  // ---- tasks ----
  // A task never lets an exception escape into the pool (a task that throws while the single-threaded pool executes it directly is queued again,
  // ThreadPool.h:451-458): the first exception of the picture is parked here, the remaining tasks of the picture finish as no-ops, and
  // waitForPrevDecompressedPic() rethrows it on the API thread — where DecLibRecon's own exceptions surface too (DecLibRecon.cpp:704-715).
  std::mutex m_failMutex; std::exception_ptr m_failure; std::atomic<bool> m_failed{ false };
  void park( std::exception_ptr e ) { std::lock_guard<std::mutex> l( m_failMutex ); if( !m_failure ) m_failure = e; m_failed.store( true ); }
  template<class F> bool guarded( F f ) { if( m_failed.load() ) return true; try { return f(); } catch( ... ) { park( std::current_exception() ); return true; } }

  // Host tasks of a picture.  MIDER: one task per CTU row that walks its CTUs as far as the row above allows — a CTU needs the CTU to its left and the CTU
  // above-right (the last one of the row: above) done, the merge / AMVP candidates of a CU reach into them (the MIDER preconditions of ctuTask,
  // DecLibRecon.cpp:764-778) — and hands itself back to the pool when it has to wait (the pool runs it again: ThreadPool.h task contract), so the wave front costs
  // one task per row, not per CTU.  FLATTEN (boundary strengths, CU / TU walk): one task per run of FLATTEN_RUN CTUs, ready when their MIDER has run; only MIDER is
  // on the wave front's critical path.  (One task per CTU — 1020 at 4K — spent more time in the pool's task scan than in the work.)
  static constexpr int FLATTEN_RUN = 3;
  struct RowTask { DecLibReconB200* self = nullptr; int line = 0; };
  struct RunTask { DecLibReconB200* self = nullptr; int line = 0, col0 = 0, col1 = 0; };
  std::vector<RowTask> m_rowTasks; std::vector<RunTask> m_runTasks; std::unique_ptr<std::atomic<int>[]> m_miderDone;      // per row: CTUs whose motion is derived
  static bool miderRowReady( int, void* p )
  {
    const RowTask& t = *static_cast<RowTask*>( p ); const DecLibReconB200& d = *t.self;
    if( d.m_failed.load() || t.line == 0 ) return true;
    const int W = d.m_ctusW, col = d.m_miderDone[t.line].load( std::memory_order_relaxed );
    return d.m_miderDone[t.line - 1].load( std::memory_order_acquire ) >= std::min( col + 2, W );
  }
  static bool miderRowTask( int tid, void* p )
  {
    RowTask& t = *static_cast<RowTask*>( p ); DecLibReconB200& d = *t.self;
    const int W = d.m_ctusW;
    int col = d.m_miderDone[t.line].load( std::memory_order_relaxed );                       // only this task advances it
    while( col < W )
    {
      if( !d.m_failed.load() && t.line > 0 && d.m_miderDone[t.line - 1].load( std::memory_order_acquire ) < std::min( col + 2, W ) ) return false;
      d.guarded( [&] { d.miderCtu( tid, d.m_rows[(size_t) t.line * W + col] ); return true; } );
      d.m_miderDone[t.line].store( ++col, std::memory_order_release );
    }
    return true;
  }
  static bool flattenRunReady( int, void* p ) { const RunTask& t = *static_cast<RunTask*>( p ); return t.self->m_failed.load() || t.self->m_miderDone[t.line].load( std::memory_order_acquire ) >= t.col1; }
  static bool flattenRunTask( int tid, void* p )
  {
    RunTask& t = *static_cast<RunTask*>( p ); DecLibReconB200& d = *t.self;
    if( !flattenRunReady( tid, p ) ) return false;
    { int64_t z = 0; d.m_tFlat0.compare_exchange_strong( z, (int64_t) ( d.since() * 1e9 ) + 1 ); }
    return d.guarded( [&] { for( int col = t.col0; col < t.col1; col++ ) d.flattenCtu( d.m_rows[(size_t) t.line * d.m_ctusW + col] ); return true; } );
  }
  void miderCtu( int tid, Row& r )
  {
    CpuTimer tm{ m_cpuNs[0] };
    CodingStructure& cs = *m_currDecompPic->cs; const PreCalcValues& pcv = *cs.pcv;
    const int a = r.line * m_ctusW + r.col;
    CtuData& cd = cs.getCtuData( a );
    cd.motion = &m_motionInfo[(size_t) pcv.num4x4CtuBlks * a];
    if( !cd.slice->isIntra() || cs.sps->getIBCFlag() ) m_cuDecoders[tid]->TaskDeriveCtuMotionInfo( cs, a, getCtuArea( cs, r.col, r.line, true ), m_hist[r.line] );
    else memset( NO_WARNING_class_memaccess( cd.motion ), MI_NOT_VALID, sizeof( MotionInfo ) * pcv.num4x4CtuBlks );
  }

  static bool finishMotionTask( int tid, void* p )
  {
    Row& r = *static_cast<Row*>( p ); DecLibReconB200& d = *r.self;
    return d.guarded( [&] {
      CodingStructure& cs = *d.m_currDecompPic->cs;
      for( int x = 0; x < d.m_ctusW; x++ ) { const int a = r.line * d.m_ctusW + x; if( !cs.getCtuData( a ).slice->isIntra() ) d.m_cuDecoders[tid]->TaskFinishMotionInfo( cs, a, x, r.line ); }
      return true; } );
  }
  // SUBMIT: ready when the pictures this one references that another recon instance is still flattening have gone into the stream
  static bool submitReady( int, void* p )
  {
    DecLibReconB200* d = static_cast<DecLibReconB200*>( p );
    if( d->m_failed.load() || d->m_waitSlots.empty() ) return true;
    std::unique_lock<std::mutex> l( d->m_sh->m, std::try_to_lock );
    if( !l.owns_lock() ) return false;
    for( int s : d->m_waitSlots ) if( d->m_sh->valid[s] == 2 ) return false;
    return true;
  }
  static bool submitTask( int, void* p ) { DecLibReconB200* d = static_cast<DecLibReconB200*>( p ); d->m_stage[2] = d->since(); const bool r = d->guarded( [&] { d->submit(); return true; } ); d->m_stage[3] = d->since(); return r; }


  void flattenCtu( Row& r )
  {
    Picture* pic = m_currDecompPic; CodingStructure& cs = *pic->cs; const SPS& sps = *cs.sps; const PreCalcValues& pcv = *cs.pcv;
    const int W = pcv.widthInCtus, W4 = ( pcv.lumaWidth + 3 ) >> 2;
    const SliceTabs* st = nullptr;                            // the tables of the slice the current CU belongs to
    auto wp = [&st]( int r0, int r1 ) { return st->wpIdx.empty() ? 0 : st->wpIdx[( r0 + 1 ) * st->wpStride + ( r1 + 1 )]; };
    r.pus.clear(); r.tus.clear(); r.coefs.clear(); r.intra.clear(); r.lfCus.clear(); r.lfTus.clear();
    {
      const int col = r.col;
      const int a = r.line * W + col;
      CtuData& cd = cs.getCtuData( a );
      // LF_INIT (DecLibRecon.cpp:808-829); with setDeviceLfDerive the device derives the grids from the CU / TU records emitted below
      if( m_lfOn )
      {
        CpuTimer tm{ m_cpuNs[1] };
        for( auto& cu : cs.traverseCUs( a ) )
        {
          b200_lf_cu q; uint32_t n = 0;
          for( auto& tu : TUTraverser( &cu.firstTU, cu.lastTU->next ) ) { b200_lf_tu t; flattenLfTu( tu, t ); r.lfTus.push_back( t ); n++; }
          flattenLfCu( cu, (uint32_t) ( r.lfTus.size() - n ), n, 0, sliceIdx( cu.slice ), q );
          r.lfCus.push_back( q );
        }
      }
      else
      {
        cd.lfParam[0] = &m_loopFilterParam[(size_t) pcv.num4x4CtuBlks * ( 2 * a )]; cd.lfParam[1] = &m_loopFilterParam[(size_t) pcv.num4x4CtuBlks * ( 2 * a + 1 )];
        memset( cd.lfParam[0], 0, sizeof( LoopFilterParam ) * 2 * pcv.num4x4CtuBlks );
        CpuTimer tm{ m_cpuNs[1] };
        m_cLoopFilter.calcFilterStrengthsCTU( cs, a );
        for( int dir = 0; dir < 2; dir++ ) flattenLfCtu( cs, a, dir, m_lf[dir].v.data() );
      }
      size_t lfCu = 0;                                        // the CU record of the current CU (records follow cs.traverseCUs like this walk)
      (void) W4;
      CpuTimer tm2{ m_cpuNs[2] };
      // the CU / TU walks of TaskTrafoCtu + TaskInterCtu + TaskCriticalIntraKernel (DecCu.cpp:106-159)
      for( auto& cu : cs.traverseCUs( a ) )
      {
        if( !st || st->slice != cu.slice ) st = &m_sl[sliceIdx( cu.slice )];
        if( m_lfOn ) r.lfCus[lfCu++].firstPu = (uint32_t) r.pus.size();
        if( CU::isIntra( cu ) )
        {
          // K6: one b200_intra_tu per TU component in decoding order (the order DecCu::predAndReco walks them, DecCu.cpp:284-288); the residual of
          // a coded component goes through K1 into the residual planes (B200_TU_RESI) and is added by K6
          if( cu.ispMode() && isLuma( cu.chType() ) )
          {
            // intra sub-partitions: K6 takes the luma as one record per prediction region (the regions read each other's reconstruction, in order), K1 the
            // residual of every sub-partition with a coded block flag — 1- and 2-sample-wide transform units included (TrQuant.cpp:466-482)
            if( flattenIspCu( cu, [&]( const b200_intra_tu& q ) { r.intra.push_back( q ); } ) != FLATTEN_INTRA_OK ) THROW_UNSUPPORTED( "DecLibReconB200: ISP CU outside the device path" );
            for( auto& tu : TUTraverser( &cu.firstTU, cu.lastTU->next ) ) { b200_tu t; if( flattenTU( tu, COMPONENT_Y, *m_trQuant, r.coefs, t ) ) { t.flags |= B200_TU_RESI; setSlOff( cu, t ); r.tus.push_back( t ); } }
          }
          for( auto& tu : TUTraverser( &cu.firstTU, cu.lastTU->next ) )
            for( const CompArea& area : tu.blocks )
            {
              if( !area.valid() ) continue;
              if( cu.ispMode() && isLuma( area.compID() ) ) continue;              // done above
              b200_intra_tu ir;
              if( flattenIntraTU( tu, area.compID(), ir ) != FLATTEN_INTRA_OK ) THROW_UNSUPPORTED( "DecLibReconB200: ACT intra block (SURVEY 8f-1)" );
              b200_tu t;
              if( flattenTU( tu, area.compID(), *m_trQuant, r.coefs, t ) ) { t.flags |= B200_TU_RESI; setSlOff( cu, t ); r.tus.push_back( t ); }
              if( TU::getCbf( tu, area.compID() ) || ( isChroma( area.compID() ) && tu.jointCbCr ) ) ir.flags |= B200_INTRA_ADD_RESI;      // DecCu.cpp:390
              r.intra.push_back( ir );
            }
          continue;
        }
        if( !CU::isInter( cu ) ) THROW_UNSUPPORTED( "DecLibReconB200: IBC CU (SURVEY 8f-1)" );
        bool ciipComp[3] = { false, false, false };
        if( cu.ciipFlag() )
        {
          // CIIP: the inter prediction comes from K2 like any merge CU; K6 blends a planar intra block into it (predBlendIntraCiip) and adds the residual
          for( int c = 0; c < (int) getNumberValidComponents( cu.chromaFormat ); c++ )
          {
            b200_intra_tu ir;
            if( flattenCiipBlock( cu, ComponentID( c ), ir ) != FLATTEN_INTRA_OK ) continue;
            if( cu.rootCbf() )                                           // (a CU larger than the maximum transform size carries several TUs under the one CIIP block)
              for( auto& tu : TUTraverser( &cu.firstTU, cu.lastTU->next ) ) if( TU::getCbf( tu, ComponentID( c ) ) || ( c && tu.jointCbCr ) ) ir.flags |= B200_INTRA_ADD_RESI;
            r.intra.push_back( ir ); ciipComp[c] = true;
          }
        }
        FlattenPuResult rc;
        if( cu.mergeType() == MRG_TYPE_SUBPU_ATMVP ) rc = flattenSbTmvp( cu, st->slotMap, wp, [&]( const b200_pu& q ) { r.pus.push_back( q ); } );
        else
        {
          b200_pu q; rc = flattenPU( cu, st->slotMap, wp, q );
          if( rc == FLATTEN_PU_OK ) { r.pus.push_back( q ); if( q.flags & B200_PU_DMVR ) cu.setDmvrCondition( true ); }   // motionCompensation :1436 sets it on the CPU path; TaskFinishMotionInfo reads it
        }
        if( rc != FLATTEN_PU_OK ) THROW_UNSUPPORTED( "DecLibReconB200: inter tool outside the device path (RPR-scaled reference, wrap-around, sub-picture clipping)" );
        if( cu.rootCbf() )
          for( auto& tu : TUTraverser( &cu.firstTU, cu.lastTU->next ) )
            for( int c = 0; c < (int) getNumberValidComponents( cu.chromaFormat ); c++ ) { b200_tu t; if( flattenTU( tu, ComponentID( c ), *m_trQuant, r.coefs, t ) ) { if( ciipComp[c] ) t.flags |= B200_TU_RESI; setSlOff( cu, t ); r.tus.push_back( t ); } }
      }
    }
  }

  // picture-level tables (slice / APS / SPS level state), before the row tasks start
  void preparePicture( Picture* pic )
  {
    CodingStructure& cs = *pic->cs; const SPS& sps = *cs.sps; const PPS& pps = *cs.pps; const PreCalcValues& pcv = *cs.pcv;
    Shared& S = *m_sh;
    {
      // A picture with another picture size / bit depth / CTU size / chroma format than the device context was built for: a new coded video sequence (new
      // parameter sets at an IRAP picture).  The pictures the other recon instances still hold are finished (their planes go back to the host, output reads those),
      // then the device context is rebuilt for this geometry.  With several threads DecLib may still hand over a picture of the OLD sequence afterwards
      // (DecLibParser::getNextDecodablePicture): the context then switches back and the references are uploaded from their host planes (importReference).
      // A REFERENCE of another size than the picture itself is reference picture resampling: refused there.
      bool changed;
      {
        std::lock_guard<std::mutex> l( S.m );
        changed = !S.owner.empty() && ( (int) pcv.lumaWidth != S.geom.width || (int) pcv.lumaHeight != S.geom.height || sps.getBitDepth() != S.geom.bitDepth
                                        || (int) pcv.maxCUWidth != S.geom.ctuSize || ( sps.getChromaFormatIdc() == CHROMA_420 ? 1 : 0 ) != S.geom.chromaFormat );
      }
      if( changed )
      {
        std::vector<DecLibReconB200*> others;
        { std::lock_guard<std::mutex> l( S.m ); others = S.instances; }
        for( DecLibReconB200* o : others ) if( o != this && o->m_currDecompPic ) o->finishCurrent();
        std::lock_guard<std::mutex> l( S.m );
        if( S.ctx ) { b200_ctx_destroy( S.ctx ); S.ctx = nullptr; }
        S.slotOf.clear(); S.owner.clear(); S.valid.clear();
      }
    }
    if( !m_fltBuf.bufs.empty() && ( m_fltFmt != pcv.chrFormat || m_fltCtu != (int) pcv.maxCUWidth ) ) m_fltBuf.destroy();
    m_fltFmt = pcv.chrFormat; m_fltCtu = (int) pcv.maxCUWidth;
    {
      std::lock_guard<std::mutex> l( S.m );
      if( !S.ctx && !m_dryRun )
      {
        S.geom.width = pcv.lumaWidth; S.geom.height = pcv.lumaHeight; S.geom.bitDepth = sps.getBitDepth(); S.geom.chromaFormat = sps.getChromaFormatIdc() == CHROMA_420 ? 1 : 0;
        S.geom.ctuSize = pcv.maxCUWidth; S.geom.stride[0] = pcv.lumaWidth; S.geom.stride[1] = S.geom.stride[2] = pcv.lumaWidth >> 1;
        S.numSlots = m_dpbSlots; S.owner.assign( S.numSlots, nullptr ); S.valid.assign( S.numSlots, 0 );
        check( b200_ctx_create( &S.ctx, &S.geom, S.numSlots, 4, -1 ) );
      }
      else if( S.owner.empty() )
      {
        S.geom.width = pcv.lumaWidth; S.geom.height = pcv.lumaHeight; S.geom.bitDepth = sps.getBitDepth(); S.geom.chromaFormat = sps.getChromaFormatIdc() == CHROMA_420 ? 1 : 0;
        S.geom.ctuSize = pcv.maxCUWidth; S.geom.stride[0] = pcv.lumaWidth; S.geom.stride[1] = S.geom.stride[2] = pcv.lumaWidth >> 1;
        S.numSlots = m_dpbSlots; S.owner.assign( S.numSlots, nullptr ); S.valid.assign( S.numSlots, 0 );
      }
      // reference pictures -> device DPB slots (uploaded if the device does not hold them)
      m_waitSlots.clear(); m_refSlots.clear();
      m_sl.assign( pic->slices.size(), SliceTabs() );
      for( size_t si = 0; si < pic->slices.size(); si++ )
      {
        const Slice& sl = *pic->slices[si]; SliceTabs& st = m_sl[si]; st.slice = &sl;
        memset( &st.slotMap, -1, sizeof( st.slotMap ) );
        for( int l = 0; l < 2; l++ ) for( int i = 0; i < sl.getNumRefIdx( RefPicList( l ) ); i++ ) { st.slotMap.slot[l][i] = (int8_t) importReference( sl.getRefPic( RefPicList( l ), i ) ); m_refSlots.push_back( st.slotMap.slot[l][i] ); }
      }
      m_slotMap = m_sl[0].slotMap;
      m_dstSlot = slotLocked( pic ); S.valid[m_dstSlot] = 2;
    }
    const Slice& slice0 = *pic->slices[0];
    // explicit weighted prediction: one entry per (refIdx0, refIdx1) combination of every slice (getWpScaling, WeightPrediction.cpp:67)
    m_wp.clear();
    for( SliceTabs& st : m_sl )
    {
      const Slice& sl = *st.slice;
      if( !( ( pps.getWPBiPred() && sl.isInterB() ) || ( pps.getUseWP() && sl.isInterP() ) ) ) continue;
      const int n0 = sl.getNumRefIdx( REF_PIC_LIST_0 ), n1 = sl.isInterB() ? sl.getNumRefIdx( REF_PIC_LIST_1 ) : 0;
      st.wpStride = n1 + 1; st.wpIdx.assign( (size_t) ( n0 + 1 ) * ( n1 + 1 ), 0 );
      for( int r0 = -1; r0 < n0; r0++ ) for( int r1 = -1; r1 < n1; r1++ )
      {
        if( r0 < 0 && r1 < 0 ) continue;
        WPScalingParam w0[3], w1[3]; WeightPrediction wpObj; wpObj.getWpScaling( &sl, r0, r1, w0, w1 );
        b200_wp e{}; const bool bi = r0 >= 0 && r1 >= 0; const WPScalingParam* u = r0 >= 0 ? w0 : w1;
        for( int c = 0; c < 3; c++ ) { e.w0[c] = bi ? w0[c].w : u[c].w; e.w1[c] = bi ? w1[c].w : 0; e.offset[c] = bi ? w0[c].offset : u[c].offset; e.shift[c] = bi ? w0[c].shift : u[c].shift; }
        m_wp.push_back( e ); st.wpIdx[( r0 + 1 ) * st.wpStride + ( r1 + 1 )] = (int) m_wp.size();
      }
    }
    if( m_wp.size() > 255 ) THROW_UNSUPPORTED( "DecLibReconB200: more than 255 weighted-prediction combinations" );
    // deblocking: slice offsets and the SPS's luma-adaptive QP offsets (deriveLADFShift, LoopFilter.cpp:1363)
    m_lfSlices.assign( m_sl.size(), b200_lf_slice{} );
    for( size_t si = 0; si < m_sl.size(); si++ )
    {
      const Slice& sl = *m_sl[si].slice; b200_lf_slice& f = m_lfSlices[si];
      f.disable = sl.getDeblockingFilterDisable();
      f.betaOffsetDiv2[0] = sl.getDeblockingFilterBetaOffsetDiv2();   f.tcOffsetDiv2[0] = sl.getDeblockingFilterTcOffsetDiv2();
      f.betaOffsetDiv2[1] = sl.getDeblockingFilterCbBetaOffsetDiv2(); f.tcOffsetDiv2[1] = sl.getDeblockingFilterCbTcOffsetDiv2();
      f.betaOffsetDiv2[2] = sl.getDeblockingFilterCrBetaOffsetDiv2(); f.tcOffsetDiv2[2] = sl.getDeblockingFilterCrTcOffsetDiv2();
    }
    m_lfSeq = b200_lf_seq{};
    if( sps.getLadfEnabled() )
    {
      m_lfSeq.ladfEnabled = 1; m_lfSeq.ladfNumIntervals = sps.getLadfNumIntervals();
      for( int k = 0; k < sps.getLadfNumIntervals() && k < 5; k++ ) { m_lfSeq.ladfQpOffset[k] = sps.getLadfQpOffset( k ); m_lfSeq.ladfIntervalLowerBound[k] = sps.getLadfIntervalLowerBound( k ); }
    }
    // explicit scaling lists (Quant::init: the first slice that uses them names the APS, Quant.cpp:623-672)
    m_useSL = false; for( const Slice* sl : pic->slices ) m_useSL = m_useSL || sl->getExplicitScalingListUsed();
    if( m_useSL )
    {
      if( !m_quant ) m_quant.reset( new Quant( nullptr ) );
      m_quant->init( pic );
      m_slBase = m_quant->getDequantCoeff( 0, 0, 0 );
      m_slCount = (size_t) ( m_quant->getDequantCoeff( SCALING_LIST_NUM - 1, SCALING_LIST_SIZE_NUM - 1, SCALING_LIST_SIZE_NUM - 1 ) - m_slBase ) + 64 * 64;
      if( m_slReg != m_slBase && !m_dryRun ) { unpinScaling(); if( b200_host_register( const_cast<int*>( m_slBase ), m_slCount * sizeof( int ) ) == 0 ) m_slReg = m_slBase; }
    }
    m_doSao = sps.getUseSAO();
    { const char* e = getenv( "B200_LF_DERIVE" ); m_lfOn = m_lfDerive || ( e && e[0] == '1' ); }
    m_doAlf = sps.getUseALF() && !AdaptiveLoopFilter::getAlfSkipPic( cs );
    const int W4 = ( pcv.lumaWidth + 3 ) >> 2, H4 = ( pcv.lumaHeight + 3 ) >> 2;
    for( int d = 0; d < 2; d++ ) { m_lf[d].v.resize( (size_t) W4 * H4 ); if( !m_lfOn || m_dryRun ) m_lf[d].pin(); }   // every entry is rewritten by flattenLfCtu (or deriveLfOnHost)
    m_sao.v.assign( pcv.sizeInCtus, b200_sao_ctu{} ); m_alf.v.assign( pcv.sizeInCtus, b200_alf_ctu{} ); m_sao.pin(); m_alf.pin();
    for( auto& s : m_sao.v ) s.type[0] = s.type[1] = s.type[2] = B200_SAO_OFF;
    if( m_doAlf )
    {
      if( m_fltBuf.bufs.empty() ) m_fltBuf.create( pcv.chrFormat, Size( 16, 16 ), pcv.maxCUWidth, 0, MEMORY_ALIGN_DEF_SIZE );
      m_cALF.create( cs.picHeader.get(), &sps, &pps, 1, m_fltBuf );              // fills m_clipDefault for the bit depth
      std::vector<const Slice*> sls; for( const SliceTabs& st : m_sl ) sls.push_back( st.slice );
      // the per-class tables (lumaCoeffFinal / lumaClippFinal / chrmClippFinal) are derived from the coded APS by the slice PARSE task (DecSlice.cpp:87), which
      // need not have run yet when DecLib hands the picture over (RECO_WHILE_PARSE): derived here if not done (idempotent, under the APS's own mutex)
      for( const Slice* sl : sls ) AdaptiveLoopFilter::reconstructCoeffAPSs( *const_cast<Slice*>( sl ) );
      std::vector<AlfSliceBase> bases;
      m_alfTabs = buildAlfTablesOfSlices( sls, &m_cALF.m_fixedFilterSetCoeffDec[0][0], m_cALF.m_clipDefault, m_alfStore, bases );
      for( size_t si = 0; si < m_sl.size(); si++ ) m_sl[si].alf = bases[si];
      if( m_alfTabs.numLumaSets > 255 || m_alfTabs.numChromaAlts > 255 || m_alfTabs.numCc[0] > 254 || m_alfTabs.numCc[1] > 254 ) THROW_UNSUPPORTED( "DecLibReconB200: more ALF sets in a picture than a CTU record can address" );
    }
    // LMCS tables (Reshape::initSlice as DecLibRecon.cpp:448-452)
    m_doLmcs = sps.getUseReshaper() && cs.picHeader->getLmcsEnabledFlag() && slice0.getLmcsEnabledFlag();
    if( m_doLmcs )
    {
      m_cReshaper.createDec( sps.getBitDepth() ); m_cReshaper.initSlice( slice0.getNalUnitLayerId(), *slice0.getPicHeader(), slice0.getVPS_nothrow() );
      m_lmcs = b200_lmcs{}; m_lmcs.chromaAdj = m_cReshaper.m_sliceReshapeInfo.enableChromaAdj;
      m_lmcs.minBinIdx = m_cReshaper.m_sliceReshapeInfo.reshaperModelMinBinIdx; m_lmcs.maxBinIdx = m_cReshaper.m_sliceReshapeInfo.reshaperModelMaxBinIdx; m_lmcs.orgCW = m_cReshaper.m_initCW;
      for( int i = 0; i < 17; i++ ) { m_lmcs.reshapePivot[i] = m_cReshaper.m_reshapePivot[i]; m_lmcs.inputPivot[i] = m_cReshaper.m_inputPivot[i]; }
      for( int i = 0; i < 16; i++ ) { m_lmcs.fwdScaleCoef[i] = m_cReshaper.m_fwdScaleCoef[i]; m_lmcs.chromaAdjHelpLUT[i] = m_cReshaper.m_chromaAdjHelpLUT[i]; }
      m_lmcs.invLUT = m_cReshaper.m_invLUT;
    }
  }

  // The device's edge derivation run on the host (dry run: no device), from the records of p into m_lf: lf_derive.cuh's serial driver, in the order the device keeps.
  std::vector<uint32_t> m_lfMap[2]; std::vector<b200::LfMi> m_lfMi;
  void deriveLfOnHost( const b200_picture& p )
  {
    const b200_geom& g = m_sh->geom; const size_t n4 = (size_t) ( g.width >> 2 ) * ( g.height >> 2 );
    for( auto& m : m_lfMap ) m.resize( n4 );
    m_lfMi.resize( n4 );
    b200::LfDerive G{};
    G.W4 = g.width >> 2; G.H4 = g.height >> 2; G.ctuSize = g.ctuSize; G.chroma = g.chromaFormat; G.qpBdOffset2 = 12 * ( g.bitDepth - 8 );
    G.cus = p.lfCus; G.tus = p.lfTus; G.pus = p.pus; G.numPus = p.numPus; G.cuMap[0] = m_lfMap[0].data(); G.cuMap[1] = m_lfMap[1].data(); G.mi = m_lfMi.data();
    G.slices = p.lfSlices; G.sliceB = p.lfSliceB; G.grid[0] = m_lf[0].v.data(); G.grid[1] = m_lf[1].v.data();
    uint32_t* const maps[2] = { m_lfMap[0].data(), m_lfMap[1].data() };
    b200::lf_derive_serial( G, maps, p.numLfCus, p.lfCtuCus, (int) m_lfCtuCus.v.size() - 1, kGeoParams );
  }

  // joins the row lists, derives the VPDU records and hands the picture to the device
  void submit()
  {
    Picture* pic = m_currDecompPic; CodingStructure& cs = *pic->cs; const PreCalcValues& pcv = *cs.pcv; const Slice& slice0 = *pic->slices[0];
    size_t nP = 0, nT = 0, nC = 0, nI = 0;
    for( const Row& r : m_rows ) { nP += r.pus.size(); nT += r.tus.size(); nC += r.coefs.size(); nI += r.intra.size(); }
    m_pus.v.resize( nP ); m_tus.v.resize( nT ); m_coefs.v.resize( nC ); m_intra.v.resize( nI );
    nP = nT = nC = nI = 0;
    for( Row& r : m_rows )
    {
      if( !r.pus.empty() ) memcpy( &m_pus.v[nP], r.pus.data(), r.pus.size() * sizeof( b200_pu ) );
      for( size_t i = 0; i < r.tus.size(); i++ ) { m_tus.v[nT + i] = r.tus[i]; m_tus.v[nT + i].coefOff += (uint32_t) nC; }
      if( !r.coefs.empty() ) memcpy( &m_coefs.v[nC], r.coefs.data(), r.coefs.size() * sizeof( int16_t ) );
      if( !r.intra.empty() ) memcpy( &m_intra.v[nI], r.intra.data(), r.intra.size() * sizeof( b200_intra_tu ) );
      nP += r.pus.size(); nT += r.tus.size(); nC += r.coefs.size(); nI += r.intra.size();
    }
    // in-loop filter parameters of every CTU (the SAO availability looks at the CTUs below: the whole picture is parsed by now)
    m_ctuSlice.v.assign( pcv.sizeInCtus, 0 ); m_ctuSlice.pin();
    if( m_doSao )
    {
      // the parser leaves SAO_MODE_MERGE entries and coded offsets: resolved the way SAOPrepareCTULine does (SampleAdaptiveOffset.cpp:400-424), in raster order,
      // with the reference's own merge candidates (left / above CTU of the same slice and tile) and offset scaling
      PelUnitBuf none;
      m_cSAO.create( pcv.lumaWidth, pcv.lumaHeight, pcv.chrFormat, pcv.maxCUWidth, pcv.maxCUHeight, 0, (uint32_t) std::max( 0, cs.sps->getBitDepth() - MAX_SAO_TRUNCATED_BITDEPTH ), none );
      for( unsigned a = 0; a < pcv.sizeInCtus; a++ )
      {
        SAOBlkParam* mergeList[NUM_SAO_MERGE_TYPES] = { nullptr, nullptr };
        m_cSAO.getMergeList( cs, (int) a, mergeList );
        m_cSAO.reconstructBlkSAOParam( cs.getCtuData( a ).saoParam, mergeList );
      }
    }
    for( unsigned a = 0; a < pcv.sizeInCtus; a++ )
    {
      CtuData& cd = cs.getCtuData( a );
      if( m_doSao )
      {
        bool av[8];
        m_cSAO.deriveLoopFilterBoundaryAvailibility( cs, Position( ( a % pcv.widthInCtus ) * pcv.maxCUWidth, ( a / pcv.widthInCtus ) * pcv.maxCUHeight ), av[0], av[1], av[2], av[3], av[4], av[5], av[6], av[7] );
        flattenSAO( cd.saoParam, av, getNumberValidComponents( pcv.chrFormat ), m_sao.v[a] );
      }
      const int si = sliceIdx( cd.slice ); m_ctuSlice.v[a] = (uint8_t) si;
      if( m_doAlf )
      {
        // CTU-level indices are relative to the slice's own APS lists: moved behind the sets of the slices before it (buildAlfTablesOfSlices)
        b200_alf_ctu& q = m_alf.v[a]; flattenALF( cd.alfParam, q );
        const Slice& sl = *cd.slice; const AlfSliceBase& ab = m_sl[si].alf;
        {
          // CTUs whose neighbours ALF may not read (in-loop filtering disabled across slices / tiles): the reference's own derivation (AdaptiveLoopFilter.cpp:118)
          bool cT, cB, cL, cR; int nH = 0, nV = 0, hp[3], vp[3], rasterPad = 0;
          const Position ctuPos( ( a % pcv.widthInCtus ) * pcv.maxCUWidth, ( a / pcv.widthInCtus ) * pcv.maxCUHeight );
          const Size ctuSize( std::min<int>( pcv.maxCUWidth, pcv.lumaWidth - ctuPos.x ), std::min<int>( pcv.maxCUHeight, pcv.lumaHeight - ctuPos.y ) );
          if( m_cALF.isClipOrCrossedByVirtualBoundaries( cs, Area( ctuPos, ctuSize ), cT, cB, cL, cR, nH, nV, hp, vp, rasterPad ) )
          {
            if( nH || nV ) THROW_UNSUPPORTED( "DecLibReconB200: a virtual boundary inside a CTU" );
            q.enable[0] |= ( cT ? B200_ALF_CLIP_TOP : 0 ) | ( cB ? B200_ALF_CLIP_BOTTOM : 0 ) | ( cL ? B200_ALF_CLIP_LEFT : 0 ) | ( cR ? B200_ALF_CLIP_RIGHT : 0 )
                         | ( ( rasterPad & 1 ) ? B200_ALF_PAD_TL : 0 ) | ( ( rasterPad & 2 ) ? B200_ALF_PAD_BR : 0 );
            if( !sl.getCcAlfCbEnabledFlag() ) q.enable[1] |= B200_ALF_PAD_WIDE;      // a chroma plane padded on its own gets the luma margin (filterCTU :794-803)
            if( !sl.getCcAlfCrEnabledFlag() ) q.enable[2] |= B200_ALF_PAD_WIDE;
          }
        }
        if( !sl.getAlfEnabledFlag( COMPONENT_Y ) ) q.enable[0] &= ~1;
        if( !sl.getAlfEnabledFlag( COMPONENT_Cb ) ) q.enable[1] &= ~1;
        if( !sl.getAlfEnabledFlag( COMPONENT_Cr ) ) q.enable[2] &= ~1;
        if( q.lumaSet >= NUM_FIXED_FILTER_SETS ) q.lumaSet = (uint8_t) ( q.lumaSet + ab.luma );
        for( int k = 0; k < 2; k++ )
        {
          q.chromaAlt[k] = (uint8_t) ( q.chromaAlt[k] + ab.chroma );
          if( !( k == 0 ? sl.getCcAlfCbEnabledFlag() : sl.getCcAlfCrEnabledFlag() ) ) q.ccIdx[k] = 0;
          else if( q.ccIdx[k] ) q.ccIdx[k] = (uint8_t) ( q.ccIdx[k] + ab.cc[k] );
        }
      }
    }
    if( m_doLmcs )
    {
      const int vs = pcv.maxCUWidth == 128 ? 64 : pcv.maxCUWidth, vW = ( pcv.lumaWidth + vs - 1 ) / vs, vH = ( pcv.lumaHeight + vs - 1 ) / vs;
      m_vpdus.v.assign( (size_t) vW * vH, b200_lmcs_vpdu{} );
      for( int j = 0; j < vH; j++ ) for( int i = 0; i < vW; i++ )
      {
        const Position tl( i * vs, j * vs );                                                     // Reshape.cpp:217-219
        const CodingUnit* cu = cs.getCU( tl, CHANNEL_TYPE_LUMA );
        const CodingUnit* above = cs.getCURestricted( cu->lumaPos().offset( 0, -1 ), *cu, CHANNEL_TYPE_LUMA, cu->ly() == tl.y ? cu : cu->above );
        const CodingUnit* left  = cs.getCURestricted( cu->lumaPos().offset( -1, 0 ), *cu, CHANNEL_TYPE_LUMA, cu->lx() == tl.x ? cu : cu->left );
        m_vpdus.v[(size_t) j * vW + i] = b200_lmcs_vpdu{ (uint16_t) cu->lx(), (uint16_t) cu->ly(), (uint8_t) ( left != nullptr ), (uint8_t) ( above != nullptr ) };
      }
      m_lmcs.vpdus = m_vpdus.v.data();
    }
    m_pus.pin(); m_tus.pin(); m_coefs.pin(); m_intra.pin();
    if( m_lfOn )
    {
      // the CU / TU records of every CTU, joined in raster order; TU and PU indices become picture-level
      size_t nCu = 0, nTu = 0; for( const Row& r : m_rows ) { nCu += r.lfCus.size(); nTu += r.lfTus.size(); }
      m_lfCus.v.resize( nCu ); m_lfTus.v.resize( nTu ); m_lfCtuCus.v.resize( m_rows.size() + 1 );
      nCu = nTu = nP = 0;
      for( size_t a = 0; a < m_rows.size(); a++ )
      {
        const Row& r = m_rows[a];
        m_lfCtuCus.v[a] = (uint32_t) nCu;
        for( size_t i = 0; i < r.lfCus.size(); i++ ) { b200_lf_cu q = r.lfCus[i]; q.firstTu += (uint32_t) nTu; q.firstPu += (uint32_t) nP; m_lfCus.v[nCu + i] = q; }
        if( !r.lfTus.empty() ) memcpy( &m_lfTus.v[nTu], r.lfTus.data(), r.lfTus.size() * sizeof( b200_lf_tu ) );
        nCu += r.lfCus.size(); nTu += r.lfTus.size(); nP += r.pus.size();
      }
      m_lfCtuCus.v[m_rows.size()] = (uint32_t) nCu;
      m_lfCus.pin(); m_lfTus.pin(); m_lfCtuCus.pin();
      m_lfSliceB.assign( m_sl.size(), 0 ); for( size_t si = 0; si < m_sl.size(); si++ ) m_lfSliceB[si] = m_sl[si].slice->isInterB() ? 1 : 0;
    }
    b200_picture& p = m_pic; p = b200_picture{};
    p.dstSlot = m_dstSlot;
    bool anyLf = false; for( const b200_lf_slice& f : m_lfSlices ) anyLf = anyLf || !f.disable;
    p.flags = ( anyLf ? B200_PIC_DEBLOCK : 0 ) | ( m_doSao ? B200_PIC_SAO : 0 ) | ( m_doAlf ? B200_PIC_ALF : 0 ) | ( m_doLmcs ? B200_PIC_LMCS : 0 );
    p.pus = m_pus.v.data(); p.numPus = m_pus.v.size(); p.numDmvr = m_dmvrMvCache.size();
    p.tus = m_tus.v.data(); p.numTus = m_tus.v.size(); p.coefs = m_coefs.v.data(); p.numCoefs = m_coefs.v.size();
    if( m_useSL ) { p.scaling = m_slBase; p.numScaling = m_slCount; }
    p.lfV = m_lf[0].v.data(); p.lfH = m_lf[1].v.data(); p.lfSlices = m_lfSlices.data(); p.numLfSlices = (int32_t) m_lfSlices.size(); p.ctuSlice = m_lfSlices.size() > 1 ? m_ctuSlice.v.data() : nullptr; p.lfSeq = &m_lfSeq;
    p.sao = m_sao.v.data(); p.vb = &m_vb; p.alf = m_alf.v.data(); p.alfTabs = &m_alfTabs;
    p.wp = m_wp.data(); p.numWp = (int32_t) m_wp.size(); p.lmcs = m_doLmcs ? &m_lmcs : nullptr;
    p.intraTus = m_intra.v.data(); p.numIntraTus = m_intra.v.size();
    if( m_lfOn )
    {
      p.lfCus = m_lfCus.v.data(); p.numLfCus = m_lfCus.v.size(); p.lfTus = m_lfTus.v.data(); p.numLfTus = m_lfTus.v.size();
      p.lfCtuCus = m_lfCtuCus.v.data(); p.lfSliceB = m_lfSliceB.data();
      if( m_dryRun ) deriveLfOnHost( p );                    // without a device the host derives the grids from the same records: the work lists keep both
      else if( p.flags & B200_PIC_DEBLOCK ) { p.flags |= B200_PIC_DERIVE_LF; p.lfV = p.lfH = nullptr; }
    }
    if( m_dryRun ) { std::lock_guard<std::mutex> l( m_sh->m ); m_sh->valid[m_dstSlot] = 3; return; }
    std::lock_guard<std::mutex> l( m_sh->m );               // two recon instances share the context: submissions are serialised (stream order = decoding order)
    for( int s : m_waitSlots ) if( m_sh->valid[s] != 1 && m_sh->valid[s] != 3 ) THROW_RECOVERABLE( "DecLibReconB200: a reference picture was not reconstructed" );
    m_arena = b200_decompress_picture( m_sh->ctx, &p );
    check( m_arena );
    m_sh->valid[m_dstSlot] = 3;
  }

public:
  DecLibReconB200() = default;
  ~DecLibReconB200() { unpinScaling(); }                  // before m_quant frees the tables: a registration must not outlive its memory
  CLASS_COPY_MOVE_DELETE( DecLibReconB200 )

  // DecLibRecon::create (DecLibRecon.cpp:127)
  void create( ThreadPool* threadPool, unsigned instanceId, bool upscaleOutputEnabled )
  {
    CHECK_FATAL( upscaleOutputEnabled, "DecLibReconB200: output upscaling is not part of the device path" );
    m_pool = threadPool; m_id = instanceId; m_numThreads = std::max( 1, threadPool ? threadPool->numThreads() : 1 );
    m_sh = sharedFor( threadPool );
    { std::lock_guard<std::mutex> l( m_sh->m ); m_sh->instances.push_back( this ); }
    m_asyncFinish = asyncFinishDefault();
#ifdef B200_GLUE_TEST_HOOKS
    m_dryRun = testHooks().dryRun;
#endif
    m_trQuant.reset( new TrQuant( &m_interPred ) );
    m_cuDecoders.clear();
    for( int i = 0; i < m_numThreads; i++ ) { m_cuDecoders.emplace_back( new DecCu ); m_cuDecoders.back()->init( nullptr, &m_interPred, nullptr, m_trQuant.get() ); }
  }
  void destroy()
  {
    if( m_sh ) { std::lock_guard<std::mutex> l( m_sh->m ); auto& v = m_sh->instances; v.erase( std::remove( v.begin(), v.end(), this ), v.end() ); }
    m_cuDecoders.clear(); m_trQuant.reset(); m_sh.reset(); m_pool = nullptr;
  }
  Picture* getCurrPic() const { return m_currDecompPic; }
  void setDpbSlots( int n ) { m_dpbSlots = n; }            // before the first picture; default 17 (MAX_NUM_REF_PICS + the current picture)
  // test hook: run every host stage and keep the work lists (flattened()), without a device
  void setDryRun( bool b ) { m_dryRun = b; }
  // Derive the deblocking grids on the device (B200_PIC_DERIVE_LF) from CU / TU records instead of calcFilterStrengthsCTU + flattenLfCtu on the host, which then
  // neither runs nor uploads them.  Default off; B200_LF_DERIVE=1 in the environment switches it on for every instance (read per picture).
  void setDeviceLfDerive( bool b ) { m_lfDerive = b; }
#ifdef B200_GLUE_TEST_HOOKS
  // Test builds only (oracle/swapped_api.cpp: the reference's DecLib compiled with this class in place of DecLibRecon, on a machine without a GPU): instances
  // start in dry-run mode and, where the device result would be fetched, hand the work lists to a callback that may fill the DMVR deltas and the picture's planes.
  struct TestHooks
  {
    bool dryRun = false; void* user = nullptr;
    void ( *picture )( void* user, const b200_picture* lists, const b200_geom* geom, int32_t* dmvrDeltas, size_t numDmvr, int16_t* const planes[3], const ptrdiff_t strides[3], int poc ) = nullptr;
    void ( *loadSlot )( void* user, int slot, const int16_t* const planes[3], const ptrdiff_t strides[3], const b200_geom* geom ) = nullptr;    // b200_ctx_load_slot_strided
  };
  static TestHooks& testHooks() { static TestHooks h; return h; }
#endif
  const b200_picture& flattened() const { return m_pic; }
  // forget one picture (its Picture object is about to be destroyed or reused: PicListManager would call this where it recycles a picture)
  void releasePicture( const Picture* pic ) { if( !m_sh ) return; std::lock_guard<std::mutex> l( m_sh->m ); auto it = m_sh->slotOf.find( pic ); if( it != m_sh->slotOf.end() ) { m_sh->owner[it->second] = nullptr; m_sh->valid[it->second] = 0; m_sh->slotOf.erase( it ); } }
  // forget every picture of the device DPB (their Picture objects are about to be destroyed: end of sequence, test harness)
  void resetDpb() { if( !m_sh ) return; std::lock_guard<std::mutex> l( m_sh->m ); m_sh->slotOf.clear(); std::fill( m_sh->owner.begin(), m_sh->owner.end(), nullptr ); std::fill( m_sh->valid.begin(), m_sh->valid.end(), 0 ); }
  const std::vector<Mv>& dmvrMvCache() const { return m_dmvrMvCache; }
  // seconds since decompressPicture(): [0] tables ready, [1] MIDER done (first flatten row starts), [2] flatten done (submit starts), [3] submitted, [4] host tasks joined, [5] device + finish done
  const double* stageTimes() const { return m_stage; }
  // CPU milliseconds of the host stages of the last picture, summed over the pool's threads: MIDER, boundary strengths + grid copy, CU / TU walk
  void cpuStageMs( double out[3] ) const { for( int i = 0; i < 3; i++ ) out[i] = m_cpuNs[i].load() * 1e-6; }

  // DecLibRecon::decompressPicture (DecLibRecon.cpp:429): schedules the host stages of the picture; returns without waiting.
  void decompressPicture( Picture* pic )
  {
    m_currDecompPic = pic;
    CodingStructure& cs = *pic->cs; const PreCalcValues& pcv = *cs.pcv;
    pic->progress = Picture::reconstructing;
    m_failure = nullptr; m_failed.store( false ); m_finished = false;
    // a picture refused here throws on the caller's thread (DecLib::reconPicture records it in pic->reconDone, DecLib.cpp:618-626); the parked copy makes
    // waitForPrevDecompressedPic() skip the picture instead of finishing work that was never scheduled
    try { refuse( pic ); finishCollocatedPictures( pic ); prepareAndSchedule( pic ); } catch( ... ) { park( std::current_exception() ); throw; }
  }
  // TMVP: MIDER reads the collocated picture's motion field (PU::getColocatedMVP -> CodingStructure::getColInfo), which TaskFinishMotionInfo writes once the
  // picture's DMVR deltas are known — for this class, when its device work has been fetched.  A collocated picture that is still with another recon instance
  // (low-delay structures: the picture decoded just before) is therefore finished here, before this picture's MIDER tasks are scheduled; DecLib's later
  // waitForPrevDecompressedPic() on that instance finds it done.
  void finishCollocatedPictures( const Picture* pic )
  {
    for( const Slice* sl : pic->slices )
    {
      if( sl->isIntra() || !sl->getPicHeader()->getEnableTMVPFlag() ) continue;
      const Picture* col = sl->getRefPic( RefPicList( sl->isInterB() ? 1 - sl->getColFromL0Flag() : 0 ), sl->getColRefIdx() );
      if( !col ) continue;
      std::vector<DecLibReconB200*> others;
      { std::lock_guard<std::mutex> l( m_sh->m ); others = m_sh->instances; }
      for( DecLibReconB200* o : others ) if( o != this && o->m_currDecompPic == col ) o->finishCurrent();
    }
  }
  void prepareAndSchedule( Picture* pic )
  {
    CodingStructure& cs = *pic->cs; const PreCalcValues& pcv = *cs.pcv;
    m_motionInfo.resize( (size_t) pcv.num4x4CtuBlks * pcv.sizeInCtus ); m_loopFilterParam.resize( (size_t) pcv.num4x4CtuBlks * pcv.sizeInCtus * 2 );
    m_dmvrMvCache.assign( (size_t) pcv.num8x8CtuBlks * pcv.sizeInCtus, Mv() ); cs.m_dmvrMvCache = m_dmvrMvCache.data();
    m_t0 = std::chrono::steady_clock::now(); m_tFlat0.store( 0 ); for( auto& c : m_cpuNs ) c.store( 0 );
    m_trQuant->init( pic );
    pic->startProcessingTimer();
    preparePicture( pic );
    m_stage[0] = since();

    const int W = pcv.widthInCtus, H = pcv.heightInCtus;
    m_ctusW = W;
    m_rows.resize( (size_t) W * H ); m_hist.assign( H, MotionHist() );
    for( int a = 0; a < W * H; a++ ) { m_rows[a].self = this; m_rows[a].line = a / W; m_rows[a].col = a % W; }
    m_miderDone.reset( new std::atomic<int>[(size_t) H] ); for( int y = 0; y < H; y++ ) m_miderDone[y].store( 0 );
    const int runsPerRow = ( W + FLATTEN_RUN - 1 ) / FLATTEN_RUN;
    m_rowTasks.assign( H, RowTask() ); m_runTasks.assign( (size_t) H * runsPerRow, RunTask() );
    pic->reconDone.lock();
    for( int y = 0; y < H; y++ )
    {
      auto bars = [&] {
        CBarrierVec b;
#if RECO_WHILE_PARSE
        if( pic->parseDone.isBlocked() ) b.push_back( &pic->ctuParsedBarrier[( y + 1 ) * W - 1] );   // the last CTU of the row is parsed (DecLibRecon.cpp:619-625)
#else
        b.push_back( &pic->parseDone );
#endif
        return b; };
      m_rowTasks[y].self = this; m_rowTasks[y].line = y;
      m_pool->addBarrierTask( TP_TASK_NAME_ARG( "POC:" + std::to_string( pic->poc ) + " b200 mider row " + std::to_string( y ) ) miderRowTask, &m_rowTasks[y], &m_flattenCounter, nullptr, bars(), miderRowReady );
      for( int k = 0; k < runsPerRow; k++ )
      {
        RunTask& t = m_runTasks[(size_t) y * runsPerRow + k]; t.self = this; t.line = y; t.col0 = k * FLATTEN_RUN; t.col1 = std::min( W, t.col0 + FLATTEN_RUN );
        m_pool->addBarrierTask( TP_TASK_NAME_ARG( "POC:" + std::to_string( pic->poc ) + " b200 flatten " + std::to_string( y ) + ":" + std::to_string( k ) ) flattenRunTask, &t, &m_flattenCounter, nullptr, bars(), flattenRunReady );
      }
    }
    m_pool->addBarrierTask( TP_TASK_NAME_ARG( "POC:" + std::to_string( pic->poc ) + " b200 submit" ) submitTask, this, &m_submitCounter, nullptr, { m_flattenCounter.donePtr(), &pic->parseDone }, submitReady );
    // FINISH as a task of its own (setAsyncFinish): the picture completes — pic->reconDone is released — without the API thread having to call
    // waitForPrevDecompressedPic() first, as the reference's finishReconTask does (DecLibRecon.cpp:663-671).  The parser relies on that when it meets a
    // decoded-picture-hash SEI with parseFrameDelay == 0 (DecLibParser.cpp:249-261: reconDone.wait() on the API thread).  The task blocks its pool thread while the device works.
    if( m_asyncFinish )
      m_pool->addBarrierTask( TP_TASK_NAME_ARG( "POC:" + std::to_string( pic->poc ) + " b200 finish" ) finishTask, this, &m_doneCounter, nullptr, { m_submitCounter.donePtr() } );
  }
  // On the device the stream orders a picture behind the pictures it references.  The test hook that stands in for the device (dry run) computes a picture when it is
  // finished: there the FINISH task only completes a picture whose references are finished and otherwise leaves it to waitForPrevDecompressedPic() (no polling: a pool
  // whose threads all found nothing ready sleeps until a task is added, ThreadPool.cpp:540-551).
  bool referencesFinished()
  {
    std::lock_guard<std::mutex> l( m_sh->m );
    for( int s : m_refSlots ) if( s >= 0 && ( m_sh->valid[s] == 2 || m_sh->valid[s] == 3 ) ) return false;
    return true;
  }
  static bool finishTask( int tid, void* p ) { static_cast<DecLibReconB200*>( p )->finishCurrent( tid ); return true; }

  // DecLibRecon::waitForPrevDecompressedPic (DecLibRecon.cpp:684): host stages done -> device done -> DMVR deltas -> TaskFinishMotionInfo -> planes.
  Picture* waitForPrevDecompressedPic()
  {
    if( !m_currDecompPic ) return nullptr;
    Picture* pic = m_currDecompPic;
    finishCurrent();
    if( m_asyncFinish ) { if( m_pool->numThreads() == 0 ) m_pool->processTasksOnMainThread(); m_doneCounter.wait_nothrow(); m_doneCounter.clearException(); }      // (the task itself, if it was not the one that finished the picture)
    m_finished = false;
    if( pic->error || pic->reconDone.hasException() ) cleanupOnException();
    return std::exchange( m_currDecompPic, nullptr );
  }
  // Completes the current picture once: from waitForPrevDecompressedPic(), from another instance that needs this picture finished (finishCollocatedPictures, change of
  // geometry), or from the FINISH task (taskTid >= 0: on a pool thread, so nothing here may wait for other pool tasks — the motion field is finished inline).
  void finishCurrent( const int taskTid = -1 )
  {
    // (the task never blocks on the mutex: whoever holds it is finishing the picture and may be waiting for pool tasks)
    std::unique_lock<std::recursive_mutex> lock( m_finishMutex, std::defer_lock );
    if( taskTid >= 0 ) { if( !lock.try_lock() ) return; } else lock.lock();
    if( m_finished ) return;
    if( taskTid >= 0 && m_dryRun && !referencesFinished() ) return;
    Picture* pic = m_currDecompPic;
    m_finished = true;
    try
    {
      if( taskTid < 0 )
      {
        if( m_pool->numThreads() == 0 ) m_pool->processTasksOnMainThread();
        m_flattenCounter.wait(); m_submitCounter.wait();
      }
      if( m_failed.load() ) std::rethrow_exception( m_failure );
      const Slice*   lastSlice           = pic->slices.back();
      const unsigned lastSliceLastCtuIdx = lastSlice->getCtuAddrInSlice( lastSlice->getNumCtuInSlice() - 1 );
      CHECK( lastSliceLastCtuIdx != pic->cs->pcv->sizeInCtus - 1, "Picture incomplete. A slice was probably lost." );
      m_stage[1] = m_tFlat0.load() * 1e-9; m_stage[4] = since();
      finishOnHost( pic, taskTid );
      m_stage[5] = since();
      if( m_failed.load() ) std::rethrow_exception( m_failure );
      pic->cs->deallocTempInternals();
      pic->stopProcessingTimer();
      pic->progress = Picture::reconstructed;
      pic->reconDone.unlock();
    }
    catch( ... )
    {
      pic->error = true;
      pic->reconDone.setException( std::current_exception() );
    }
  }
  // Completion without the API thread (see prepareAndSchedule); before the first picture.
  void setAsyncFinish( bool b ) { m_asyncFinish = b; }
  static bool& asyncFinishDefault() { static bool b = false; return b; }

  // DecLibRecon::cleanupOnException (DecLibRecon.cpp:724): no task of the broken picture may survive in the pool; its device slot is released
  void cleanupOnException()
  {
    m_flattenCounter.wait_nothrow(); m_submitCounter.wait_nothrow(); m_finishCounter.wait_nothrow(); m_doneCounter.wait_nothrow();
    m_flattenCounter.clearException(); m_submitCounter.clearException(); m_finishCounter.clearException(); m_doneCounter.clearException();
    if( m_currDecompPic ) m_currDecompPic->waitForAllTasks();
    if( m_sh && m_currDecompPic )
    {
      std::lock_guard<std::mutex> l( m_sh->m );
      auto it = m_sh->slotOf.find( m_currDecompPic );
      if( it != m_sh->slotOf.end() ) { m_sh->owner[it->second] = nullptr; m_sh->valid[it->second] = 0; m_sh->slotOf.erase( it ); }
    }
  }

private:
  void finishOnHost( Picture* pic, const int taskTid = -1 )
  {
    CodingStructure& cs = *pic->cs; const PreCalcValues& pcv = *cs.pcv; Shared& S = *m_sh;
    m_dmvr.v.assign( m_dmvrMvCache.size() * 2, 0 ); m_dmvr.pin();
    if( !m_dryRun )
    {
      std::lock_guard<std::mutex> l( S.m );
      check( b200_wait_picture( S.ctx, m_arena, m_dmvr.v.data(), m_dmvrMvCache.size() ) );
      S.valid[m_dstSlot] = 1;
    }
#ifdef B200_GLUE_TEST_HOOKS
    else if( testHooks().picture )
    {
      int16_t* planes[3] = { nullptr, nullptr, nullptr }; ptrdiff_t strides[3] = { 0, 0, 0 };
      for( int c = 0; c < ( S.geom.chromaFormat ? 3 : 1 ); c++ ) { PelBuf b = cs.getRecoBuf( ComponentID( c ) ); planes[c] = b.buf; strides[c] = b.stride; }
      testHooks().picture( testHooks().user, &m_pic, &S.geom, m_dmvr.v.data(), m_dmvrMvCache.size(), planes, strides, pic->poc );
    }
#endif
    if( m_dryRun ) { std::lock_guard<std::mutex> l( S.m ); S.valid[m_dstSlot] = 1; }
    for( size_t i = 0; i < m_dmvrMvCache.size(); i++ ) m_dmvrMvCache[i] = Mv( m_dmvr.v[2 * i], m_dmvr.v[2 * i + 1] );
    if( pic->stillReferenced && taskTid >= 0 )                                                                    // (inside the FINISH task: inline, a task must not wait for tasks)
    {
      for( unsigned a = 0; a < pcv.sizeInCtus; a++ ) if( !cs.getCtuData( a ).slice->isIntra() ) m_cuDecoders[taskTid]->TaskFinishMotionInfo( cs, a, a % pcv.widthInCtus, a / pcv.widthInCtus );
    }
    else if( pic->stillReferenced )                                                                               // colMotion for later TMVP (DecCu.cpp:161), under ctuTask's
    {                                                                                                             // conditions (DecLibRecon.cpp:860-867); one pool task per CTU row
      for( unsigned y = 0; y < pcv.heightInCtus; y++ )
        m_pool->addBarrierTask( TP_TASK_NAME_ARG( "POC:" + std::to_string( pic->poc ) + " b200 finishMotion " + std::to_string( y ) ) finishMotionTask, &m_rows[(size_t) y * pcv.widthInCtus], &m_finishCounter );
      if( m_pool->numThreads() == 0 ) m_pool->processTasksOnMainThread();
    }
    if( m_dryRun ) { m_finishCounter.wait(); return; }
    // the finished planes go back into Picture::m_bufs: output frames alias them (vvdecimpl.cpp:1051) and a CPU fallback picture may reference them
    int16_t* planes[3] = { nullptr, nullptr, nullptr }; ptrdiff_t strides[3] = { 0, 0, 0 };
    for( int c = 0; c < ( S.geom.chromaFormat ? 3 : 1 ); c++ ) { PelBuf b = cs.getRecoBuf( ComponentID( c ) ); planes[c] = b.buf; strides[c] = b.stride; }
    {
      std::lock_guard<std::mutex> l( S.m );
      check( b200_get_frame_strided( S.ctx, m_dstSlot, planes, strides ) );       // the copy runs while the pool finishes the motion field
    }
    m_finishCounter.wait();
  }
};

}   // namespace b200glue
