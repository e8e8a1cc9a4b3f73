// flatten_filters.h — host-side flatteners for the in-loop filter stages: CtuData -> b200_sao_ctu / b200_alf_ctu, APS -> b200_alf_tables,
// LoopFilterParam grids -> picture rasters.  Glue that lives INSIDE a VVdeC build; no pixel arithmetic.
// Pinned by tests/test_flatten_filters_vs_ref.py (round trip through the reference structures the shim fills for the real filters).
#pragma once
#include <vector>
#include <string.h>
#include "vvdec_b200.h"
#include "CommonLib/CommonDef.h"
#include "CommonLib/CodingStructure.h"
#include "CommonLib/Slice.h"
#include "CommonLib/SampleAdaptiveOffset.h"
#include "CommonLib/AdaptiveLoopFilter.h"

namespace b200glue
{
using namespace vvdec;

// SAOBlkParam after reconstructBlkSAOParam (merge resolved: modeIdc is NEW or OFF, SampleAdaptiveOffset.cpp:624) + the 8 availabilities of
// deriveLoopFilterBoundaryAvailibility (:741) in the order L, R, A, B, AL, AR, BL, BR.
inline void flattenSAO( const SAOBlkParam& bp, const bool avail[8], const int numComp, b200_sao_ctu& r )
{
  memset( &r, 0, sizeof( r ) );
  for( int c = 0; c < 3; c++ )
  {
    r.type[c] = B200_SAO_OFF;
    if( c >= numComp || bp[c].modeIdc == SAO_MODE_OFF ) continue;
    r.type[c] = (uint8_t) bp[c].typeIdc;                                     // SAO_TYPE_EO_0..EO_45 = 0..3, SAO_TYPE_BO = 4 (B200_SAO_* keep the values)
    if( bp[c].typeIdc == SAO_TYPE_BO )
    {
      r.band[c] = (uint8_t) bp[c].typeAuxInfo;
      for( int i = 0; i < 4; i++ ) r.offset[c][i] = (int8_t) bp[c].offset[( bp[c].typeAuxInfo + i ) & 31];   // offsetCTU :661 reads the 4 bands from the start band
    }
    else for( int i = 0; i < 5; i++ ) r.offset[c][i] = (int8_t) bp[c].offset[i];
  }
  static const uint8_t bit[8] = { B200_AVAIL_L, B200_AVAIL_R, B200_AVAIL_A, B200_AVAIL_B, B200_AVAIL_AL, B200_AVAIL_AR, B200_AVAIL_BL, B200_AVAIL_BR };
  for( int i = 0; i < 8; i++ ) if( avail[i] ) r.avail |= bit[i];
}

// CtuAlfData (CodingStructure.h:75).  alfCtbFilterIndex already is "fixed set 0..15, else 16 + position in the slice's luma APS list"
// (AdaptiveLoopFilter.cpp:509-520), which is how b200_alf_tables orders its luma sets.
inline void flattenALF( const CtuAlfData& a, b200_alf_ctu& r )
{
  memset( &r, 0, sizeof( r ) );
  for( int c = 0; c < 3; c++ ) r.enable[c] = a.alfCtuEnableFlag[c] & 1;
  r.lumaSet = (uint8_t) a.alfCtbFilterIndex;
  for( int c = 0; c < 2; c++ ) { r.chromaAlt[c] = a.alfCtuAlternative[c]; r.ccIdx[c] = a.ccAlfFilterControl[c]; }
}

// The coefficient / clipping tables of one slice: 16 fixed sets (AdaptiveLoopFilter::m_fixedFilterSetCoeffDec / m_clipDefault), then the
// slice's luma APSs in list order (lumaCoeffFinal / lumaClippFinal, reconstructCoeffAPSs :335), the chroma APS's alternatives and the
// CC-ALF filters.  `store` owns the memory the returned struct points into (pin it once: the tables change per slice at most).
struct AlfTableStore { std::vector<int16_t> lumaCoeff, lumaClip, chromaCoeff, chromaClip, cc[2]; };
// Several slices: every slice's sets go behind the ones before it; `bases` receives, per slice, what has to be added to the CTU-level indices of its CTUs
// (luma sets >= 16, chroma alternatives, CC-ALF filter numbers 1..n) so that they address the picture-level tables.
struct AlfSliceBase { int luma = 0, chroma = 0, cc[2] = { 0, 0 }; };
inline b200_alf_tables buildAlfTablesOfSlices( const std::vector<const Slice*>& slices, const short* fixedSetCoeffDec, const short* clipDefault, AlfTableStore& store, std::vector<AlfSliceBase>& bases )
{
  constexpr int SET = MAX_NUM_ALF_TRANSPOSE_ID * MAX_NUM_ALF_CLASSES * MAX_NUM_ALF_LUMA_COEFF;
  store.lumaCoeff.assign( (size_t) NUM_FIXED_FILTER_SETS * SET, 0 ); store.lumaClip.assign( store.lumaCoeff.size(), 0 );
  memcpy( store.lumaCoeff.data(), fixedSetCoeffDec, sizeof( int16_t ) * NUM_FIXED_FILTER_SETS * SET );
  for( int i = 0; i < NUM_FIXED_FILTER_SETS * SET; i++ ) store.lumaClip[i] = clipDefault[i % MAX_NUM_ALF_LUMA_COEFF];
  store.chromaCoeff.clear(); store.chromaClip.clear(); store.cc[0].clear(); store.cc[1].clear();
  bases.assign( slices.size(), AlfSliceBase() );
  b200_alf_tables t; memset( &t, 0, sizeof( t ) );
  int nLuma = 0;
  for( size_t s = 0; s < slices.size(); s++ )
  {
    const Slice& slice = *slices[s]; const APS* const* apss = slice.getAlfAPSs();
    bases[s].luma = nLuma; bases[s].chroma = t.numChromaAlts; bases[s].cc[0] = t.numCc[0]; bases[s].cc[1] = t.numCc[1];
    if( slice.getAlfEnabledFlag( COMPONENT_Y ) )
      for( int i = 0; i < slice.getNumAlfAps(); i++, nLuma++ )
      {
        const AlfSliceParam& p = apss[slice.getAlfApsIdsLuma()[i]]->getAlfAPSParam();
        store.lumaCoeff.insert( store.lumaCoeff.end(), p.lumaCoeffFinal, p.lumaCoeffFinal + SET ); store.lumaClip.insert( store.lumaClip.end(), p.lumaClippFinal, p.lumaClippFinal + SET );
      }
    if( slice.getAlfEnabledFlag( COMPONENT_Cb ) || slice.getAlfEnabledFlag( COMPONENT_Cr ) )
    {
      const AlfSliceParam& p = apss[slice.getAlfApsIdChroma()]->getAlfAPSParam();
      for( int a = 0; a < p.numAlternativesChroma; a++ )
        for( int k = 0; k < MAX_NUM_ALF_CHROMA_COEFF; k++ ) { store.chromaCoeff.push_back( p.chromaCoeff[a * MAX_NUM_ALF_CHROMA_COEFF + k] ); store.chromaClip.push_back( p.chrmClippFinal[a * MAX_NUM_ALF_CHROMA_COEFF + k] ); }
      t.numChromaAlts += p.numAlternativesChroma;
    }
    for( int c = 0; c < 2; c++ )
      if( c == 0 ? slice.getCcAlfCbEnabledFlag() : slice.getCcAlfCrEnabledFlag() )
      {
        const CcAlfFilterParam& cp = apss[c == 0 ? slice.getCcAlfCbApsId() : slice.getCcAlfCrApsId()]->getCcAlfAPSParam();
        for( int f = 0; f < cp.ccAlfFilterCount[c]; f++ ) for( int k = 0; k < 7; k++ ) store.cc[c].push_back( cp.ccAlfCoeff[c][f][k] );
        t.numCc[c] += cp.ccAlfFilterCount[c];
      }
  }
  t.lumaCoeff = store.lumaCoeff.data(); t.lumaClip = store.lumaClip.data(); t.numLumaSets = NUM_FIXED_FILTER_SETS + nLuma;
  t.chromaCoeff = store.chromaCoeff.data(); t.chromaClip = store.chromaClip.data(); t.ccCoeff[0] = store.cc[0].data(); t.ccCoeff[1] = store.cc[1].data();
  return t;
}

inline b200_alf_tables buildAlfTables( const Slice& slice, const short* fixedSetCoeffDec /* [16][1300] */, const short* clipDefault /* [13] */, AlfTableStore& store )
{
  constexpr int SET = MAX_NUM_ALF_TRANSPOSE_ID * MAX_NUM_ALF_CLASSES * MAX_NUM_ALF_LUMA_COEFF;   // 4 * 25 * 13
  const int numAps = slice.getNumAlfAps();
  store.lumaCoeff.assign( (size_t) ( NUM_FIXED_FILTER_SETS + numAps ) * SET, 0 ); store.lumaClip.assign( store.lumaCoeff.size(), 0 );
  memcpy( store.lumaCoeff.data(), fixedSetCoeffDec, sizeof( int16_t ) * NUM_FIXED_FILTER_SETS * SET );
  for( int i = 0; i < NUM_FIXED_FILTER_SETS * SET; i++ ) store.lumaClip[i] = clipDefault[i % MAX_NUM_ALF_LUMA_COEFF];
  const APS* const* apss = slice.getAlfAPSs();
  for( int i = 0; i < numAps; i++ )
  {
    const AlfSliceParam& p = apss[slice.getAlfApsIdsLuma()[i]]->getAlfAPSParam();
    memcpy( store.lumaCoeff.data() + (size_t) ( NUM_FIXED_FILTER_SETS + i ) * SET, p.lumaCoeffFinal, sizeof( int16_t ) * SET );
    memcpy( store.lumaClip.data()  + (size_t) ( NUM_FIXED_FILTER_SETS + i ) * SET, p.lumaClippFinal, sizeof( int16_t ) * SET );
  }
  b200_alf_tables t; memset( &t, 0, sizeof( t ) );
  t.lumaCoeff = store.lumaCoeff.data(); t.lumaClip = store.lumaClip.data(); t.numLumaSets = NUM_FIXED_FILTER_SETS + numAps;
  store.chromaCoeff.clear(); store.chromaClip.clear();
  if( slice.getAlfEnabledFlag( COMPONENT_Cb ) || slice.getAlfEnabledFlag( COMPONENT_Cr ) )
  {
    const AlfSliceParam& p = apss[slice.getAlfApsIdChroma()]->getAlfAPSParam();
    for( int a = 0; a < p.numAlternativesChroma; a++ )
      for( int k = 0; k < MAX_NUM_ALF_CHROMA_COEFF; k++ ) { store.chromaCoeff.push_back( p.chromaCoeff[a * MAX_NUM_ALF_CHROMA_COEFF + k] ); store.chromaClip.push_back( p.chrmClippFinal[a * MAX_NUM_ALF_CHROMA_COEFF + k] ); }
    t.numChromaAlts = p.numAlternativesChroma;
  }
  t.chromaCoeff = store.chromaCoeff.data(); t.chromaClip = store.chromaClip.data();
  for( int c = 0; c < 2; c++ )
  {
    store.cc[c].clear();
    const bool on = c == 0 ? slice.getCcAlfCbEnabledFlag() : slice.getCcAlfCrEnabledFlag();
    if( on )
    {
      const CcAlfFilterParam& cp = apss[c == 0 ? slice.getCcAlfCbApsId() : slice.getCcAlfCrApsId()]->getCcAlfAPSParam();
      const int n = cp.ccAlfFilterCount[c];
      for( int f = 0; f < n; f++ ) for( int k = 0; k < 7; k++ ) store.cc[c].push_back( cp.ccAlfCoeff[c][f][k] );
      t.numCc[c] = n;
    }
    t.ccCoeff[c] = store.cc[c].data();
  }
  return t;
}

// LoopFilterParam is 6 bytes and b200_lf_param has the same layout (static_assert below): the per-CTU arrays ctuData.lfParam[dir]
// (4x4 units in CTU raster order, stride = CTU width / 4) become rows of the picture raster.
static_assert( sizeof( LoopFilterParam ) == sizeof( b200_lf_param ), "b200_lf_param must stay byte-identical to LoopFilterParam" );
inline void flattenLfCtu( const CodingStructure& cs, const int ctuRsAddr, const int dir, b200_lf_param* raster /* [H4][W4] */ )
{
  const PreCalcValues& pcv = *cs.pcv;
  const int W4 = ( pcv.lumaWidth + 3 ) >> 2, H4 = ( pcv.lumaHeight + 3 ) >> 2, c4 = pcv.maxCUWidth >> 2;
  const int x0 = ( ctuRsAddr % pcv.widthInCtus ) * c4, y0 = ( ctuRsAddr / pcv.widthInCtus ) * c4;
  const LoopFilterParam* src = cs.getCtuData( ctuRsAddr ).lfParam[dir];
  const int w = std::min( c4, W4 - x0 ), h = std::min( c4, H4 - y0 );
  for( int y = 0; y < h; y++ ) memcpy( raster + (size_t) ( y0 + y ) * W4 + x0, src + (size_t) y * c4, sizeof( b200_lf_param ) * w );
}

// The records of the device edge derivation (B200_PIC_DERIVE_LF) in place of calcFilterStrengthsCTU + flattenLfCtu.  One b200_lf_cu per CU, in cs.traverseCUs
// order; firstTu / firstPu are where its TU records (flattenLfTu, every TU of the CU) and its first PU record go.  leftEdge / topEdge are
// LoopFilter::xGetLoopfilterParam's (LoopFilter.cpp:1063), which needs the slice and tile membership only the host has.
static_assert( sizeof( b200_lf_cu ) == 24 && sizeof( b200_lf_tu ) == 16, "b200_lf_cu / b200_lf_tu sizes are part of the C ABI" );
inline void flattenLfCu( const CodingUnit& cu, const uint32_t firstTu, const uint32_t numTus, const uint32_t firstPu, const int sliceIdx, b200_lf_cu& r )
{
  memset( &r, 0, sizeof( r ) );
  const ChannelType ch = cu.chType(); const CompArea& a = cu.blocks[ch];
  const PPS& pps = *cu.pps; const SPS& sps = *cu.sps;
  r.x = (uint16_t) a.x; r.y = (uint16_t) a.y; r.w = (uint8_t) a.width; r.h = (uint8_t) a.height;
  r.chType = (uint8_t) ch; r.treeType = (uint8_t) cu.treeType();
  uint16_t f = 0;
  if( CU::isIntra( cu ) ) f |= B200_LF_CU_INTRA;
  if( cu.ciipFlag() ) f |= B200_LF_CU_CIIP;
  if( cu.affineFlag() ) f |= B200_LF_CU_AFFINE;
  if( cu.mergeFlag() && cu.mergeType() == MRG_TYPE_SUBPU_ATMVP ) f |= B200_LF_CU_SBTMVP;
  if( cu.geoFlag() ) f |= B200_LF_CU_GEO;
  if( cu.ispMode() ) f |= B200_LF_CU_ISP;
  if( cu.bdpcmMode() ) f |= B200_LF_CU_BDPCM_Y;
  if( cu.bdpcmModeChroma() ) f |= B200_LF_CU_BDPCM_C;
  if( CU::isSepTree( cu ) ) f |= B200_LF_CU_SEP_TREE;
  auto avail = [&]( const Position p ) {
    const CodingUnit* n = cu.cs->getCU( p, ch );
    const bool sub = !sps.getSubPicInfoPresentFlag() || ( pps.getSubPicFromCU( cu ).getloopFilterAcrossSubPicEnabledFlag() && pps.getSubPicFromCU( *n ).getloopFilterAcrossSubPicEnabledFlag() );
    return CU::isAvailable( cu, *n, !pps.getLoopFilterAcrossSlicesEnabledFlag(), !pps.getLoopFilterAcrossTilesEnabledFlag(), !sub );
  };
  if( a.x > 0 && avail( a.pos().offset( -1, 0 ) ) ) f |= B200_LF_CU_AVAIL_LEFT;
  if( a.y > 0 && avail( a.pos().offset( 0, -1 ) ) ) f |= B200_LF_CU_AVAIL_TOP;
  r.flags = f;
  r.qp = (int8_t) cu.qp; r.slice = (uint8_t) sliceIdx;
  if( cu.geoFlag() ) r.geoLists = (uint8_t) ( ( ( cu.interDirrefIdxGeo0() >> 4 ) == 2 ? 1 : 0 ) | ( ( cu.interDirrefIdxGeo1() >> 4 ) == 2 ? 2 : 0 ) );
  r.numTus = (uint8_t) numTus; r.firstTu = firstTu; r.firstPu = firstPu;
}
inline void flattenLfTu( const TransformUnit& tu, b200_lf_tu& r )
{
  memset( &r, 0, sizeof( r ) );
  const CompArea& y = tu.blocks[COMPONENT_Y];
  r.x = (uint16_t) y.x; r.y = (uint16_t) y.y; r.w = (uint8_t) y.width; r.h = (uint8_t) y.height;
  if( tu.blocks.size() > 1 ) { const CompArea& c = tu.blocks[COMPONENT_Cb]; r.cx = (uint16_t) c.x; r.cy = (uint16_t) c.y; r.cw = (uint8_t) c.width; r.ch = (uint8_t) c.height; }
  r.cbf = tu.cbf; r.jointCbCr = tu.jointCbCr; r.chromaQp[0] = tu.chromaQp[0]; r.chromaQp[1] = tu.chromaQp[1];
}

}   // namespace b200glue
