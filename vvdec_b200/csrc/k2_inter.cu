// k2_inter.cu — K2: inter prediction. One CTA (256 threads) per <=16x16 luma tile of a PU (+ its two 8x8 chroma tiles):
// the reference windows of both lists are staged in shared memory (coordinates clamped to the picture = the reference's
// 144-sample border extension, Picture.cpp:400), filtered separably (8-tap luma / 4-tap chroma, 14-bit intermediates),
// then combined: rounding (uni), average / BCW (bi), BDOF, or — for DMVR tiles — a 25-point bilinear SAD search with
// parametric sub-pel refinement followed by the final MC from the padded window.  Affine PUs use a second kernel with
// one 4x4 sub-block per 16 threads (6-tap filters, PROF).  16x16 is the BDOF / DMVR processing unit of the standard,
// so tiles are independent.
//
// Where a reference position lands is decided in three places only: RefView (the clamped per-sample read), stage_windows (the
// word-wide copy of an interior footprint) and the interior predicates of its two callers (stage A in mc_tile, the search windows in
// dmvr_search).  A new rule for the reference position (wrap-around, sub-picture bounds) goes there and nowhere else.  Every stored
// sample goes through mc_sample; the shared-memory carve-up of a translational tile is tile_layout.
//
// Replaces (reference, source/Lib/CommonLib/InterPrediction.cpp): motionCompensation :1372, xPredInterBi :686, xPredInterUni :623,
// xPredInterBlk :750, xSubPuBio :551, applyBiOptFlow :1290, BiOptFlowCore :162, gradFilterCore :212, PaddBIOCore :269,
// xProcessDMVR :1847, xinitMC :1804, xBIPMVRefine :1702, xDMVRSubPixelErrorSurface :1785, xSubPelErrorSrfc :1647,
// xPrefetchPad :1525, xFinalPaddedMCForDMVR :1731, xPredAffineBlk :934, applyPROFCore :61, xWeightedAverage :1346;
// InterpolationFilter.cpp filter<> :556, filterCopy :424, filterWxH_N4/N8 :805,:881; Buffer.cpp addAvg :441, addWeightedAvg :372;
// RdCost.cpp xGetSAD8/16(+X5) :107-221; Mv.cpp clipMvInPic :64; UnitTools.cpp PU::setAllAffineMv :2689.
// HBM traffic per bi-predicted 16x16 tile: 2*(23*23 + 2*11*11)*2 B read + (256 + 128)*2 B written + 64 B record share.
#define VVC_TABLE_QUAL static __device__ const __align__(16)
#include "vvc_tables.h"
#include "common.cuh"
#include "affine_mv.cuh"
#include <algorithm>

namespace b200 {

constexpr int IFO = 8192;   // IF_INTERNAL_OFFS

struct McParams {
  int16_t* dst[3]; int dstStride[3];
  const int16_t* refs[B200_MAX_SLOTS * 3];   // device plane pointers, by value (no table in memory -> no sync when the DPB mapping changes)
  int refStride[3];
  int W, H, bitDepth, ctuSize, chroma;
  int fastOk;                                // plane strides are even -> rows are word-addressable
  const b200_pu* pus; const uint32_t* tiles; const int* meta;   // device lists (bucket.cu)
  int32_t* dmvrMv;
  const b200_wp* wp;                         // explicit weighted prediction entries (b200_pu::wpIdx), or null
  const b200_lmcs* lmcs; int lmcsLog2;       // LMCS: luma predictions are stored forward-mapped (DecCu.cpp:458-476); null = off
};

// One reference plane seen through an inclusive clamp rectangle: a position outside it reads the nearest sample inside.  The rectangle is
// the picture (the reference's border extension) or, for DMVR's final MC, the padded window intersected with the picture (xPrefetchPad
// :1525).  Every per-sample reference read goes through here, on the read-only path.
struct Rect { int x0, x1, y0, y1; };
struct RefView {
  const int16_t* p; int stride; Rect r;
  __device__ __forceinline__ int cx(int x) const { return min(max(x, r.x0), r.x1); }
  __device__ __forceinline__ int ld(int xc, int y) const { return __ldg(p + (size_t)min(max(y, r.y0), r.y1) * stride + xc); }   // xc from cx()
  __device__ __forceinline__ int at(int x, int y) const { return ld(cx(x), y); }
};

__device__ __forceinline__ void clip_mv(int& mx, int& my, int x, int y, const McParams& P)
{
  mx = clip3((-P.ctuSize - 8 - x + 1) * 16, (P.W + 8 - x - 1) * 16, mx);
  my = clip3((-P.ctuSize - 8 - y + 1) * 16, (P.H + 8 - y - 1) * 16, my);
}

__device__ __forceinline__ const int8_t* luma_taps(int frac, bool is4x4, bool altHpel)
{
  if (is4x4) return kIfLuma4x4 + frac * 8;
  if (frac == 8 && altHpel) return kIfAltHpel;
  return kIfLuma + frac * 8;
}

__device__ __forceinline__ void load_taps8(const int8_t* t, int f[8])   // rows of the tables are 8-byte aligned
{
  const int2 w = __ldg(reinterpret_cast<const int2*>(t));
#pragma unroll
  for (int k = 0; k < 4; k++) { f[k] = (w.x << (24 - 8 * k)) >> 24; f[4 + k] = (w.y << (24 - 8 * k)) >> 24; }
}

__device__ __forceinline__ int avg_bi(int p0, int p1, int w1, int hr, int pmax)
{
  int v;
  if (w1 == 4) v = (p0 + p1 + (1 << hr) + 2 * IFO) >> (hr + 1);
  else         v = (p0 * (8 - w1) + p1 * w1 + (1 << (hr + 2)) + (IFO << 3)) >> (hr + 3);
  return clip3(0, pmax, v);
}

// explicit weighted prediction (WeightPrediction.cpp:164 addWeightBi / :238 addWeightUni) on 14-bit intermediates
__device__ __forceinline__ int wp_uni(const b200_wp* e, int comp, int p, int hr, int pmax)
{
  const int s = e->shift[comp] + hr;
  return clip3(0, pmax, ((e->w0[comp] * (p + IFO) + (s > 0 ? 1 << (s - 1) : 0)) >> s) + e->offset[comp]);
}
__device__ __forceinline__ int wp_bi(const b200_wp* e, int comp, int p0, int p1, int hr, int pmax)
{
  const int s = e->shift[comp] + hr;
  return clip3(0, pmax, (e->w0[comp] * (p0 + IFO) + e->w1[comp] * (p1 + IFO) + ((1 << s) >> 1) + e->offset[comp] * (1 << (s - 1))) >> s);
}

// GEO blending weight of sample (x, y) of component scale sc in a CU of 2^l2w x 2^l2h luma samples (xWeightedGeoBlk, InterpolationFilter.cpp:1217)
__device__ __forceinline__ int geo_weight(int splitDir, int l2w, int l2h, int x, int y, int sc)
{
  const int angle = kGeoParams[splitDir * 2], mir = kGeoAngle2Mirror[angle];
  const int16_t* wo = &kGeoWeightOffset[((splitDir * 4 + (l2h - 3)) * 4 + (l2w - 3)) * 2];
  const int row = mir == 2 ? VVC_GEO_MASK_SIZE - 1 - wo[1] - (y << sc) : wo[1] + (y << sc);
  const int col = mir == 1 ? VVC_GEO_MASK_SIZE - 1 - wo[0] - (x << sc) : wo[0] + (x << sc);
  return kGeoWeights[(kGeoAngle2Mask[angle] * VVC_GEO_MASK_SIZE + row) * VVC_GEO_MASK_SIZE + col];
}
__device__ __forceinline__ int geo_blend(int wt, int p0, int p1, int hr, int pmax)
{
  const int s = hr + 3;
  return clip3(0, pmax, (wt * p0 + (8 - wt) * p1 + (1 << (s - 1)) + (IFO << 3)) >> s);
}

// final luma prediction sample -> what is stored (identity without LMCS)
__device__ __forceinline__ int luma_out(const McParams& P, int v, int pmax) { return P.lmcs ? lmcs_fwd(P.lmcs, P.lmcsLog2, v, pmax) : v; }

// What mc_sample combines: two lists' 14-bit predictions p0, p1; one list's full-precision vertical sum p0 (uni rounding takes it in one step,
// as the reference's last filter stage does); or one list's 14-bit prediction p0 (PROF).
enum McIn { MC_BI14, MC_UNI_SUM, MC_UNI14 };

// The stored sample of component comp (0 = luma, forward-mapped by LMCS) (xWeightedAverage :1346): GEO blend (geoWt >= 0), explicit WP,
// bi average / BCW (weight w1 of list 1, 4 = plain average) or uni rounding.
__device__ __forceinline__ int mc_sample(const McParams& P, int comp, McIn in, const b200_wp* we, int geoWt, int w1, int p0, int p1, int hr, int pmax)
{
  int v;
  if (geoWt >= 0)          v = geo_blend(geoWt, p0, p1, hr, pmax);
  else if (we)             v = in == MC_BI14 ? wp_bi(we, comp, p0, p1, hr, pmax) : wp_uni(we, comp, in == MC_UNI_SUM ? (int16_t)(p0 >> 6) : p0, hr, pmax);
  else if (in == MC_BI14)  v = avg_bi(p0, p1, w1, hr, pmax);
  else if (in == MC_UNI_SUM) v = clip3(0, pmax, (p0 + (1 << (5 + hr)) + (IFO << 6)) >> (6 + hr));
  else            v = clip3(0, pmax, (int)(int16_t)((p0 + (1 << (hr - 1)) + IFO) >> hr));
  return comp == 0 ? luma_out(P, v, pmax) : v;
}

__device__ __forceinline__ int shift_msb(int numer, int denom) { return numer >> (31 - __clz(denom)); }   // rightShiftMSB (:92), denom > 0

__device__ int div_for_maxq7(long long N, long long D)
{
  int sign = 0, q = 0;
  if (N < 0) { sign = 1; N = -N; }
  D <<= 3;
  if (N >= D) { N -= D; q++; }
  q <<= 1; D >>= 1;
  if (N >= D) { N -= D; q++; }
  q <<= 1;
  if (N >= (D >> 1)) q++;
  return sign ? -q : q;
}

// ------------------------------------------------------------------------------------------------ translational tiles (+BDOF, DMVR)
// MODE: 0 uni, 1 bi (average / BCW), 2 bi + BDOF, 3 DMVR (+BDOF per sub-block).  blockDim.x = tw*th (32..256): one thread per luma
// sample; tw, th are powers of two (4, 8, 16), so all index arithmetic is shifts.  Dynamic shared memory, laid out by tile_layout.
struct TileSmem {
  int16_t *w[2], *h[2];           // luma window (stride tw+8) and H-filtered rows (stride tw) per list
  int16_t *cw[2][2], *chf[2][2];  // chroma [list][comp]: window (stride cw+4), H-filtered rows (stride cw)
  int16_t *p[2];                  // BDOF: 14-bit predictions with ring (stride 18)
};

constexpr int HS = 16, CHS = 8;   // constant row strides of the H-filtered arrays (luma / chroma): column walks use immediate offsets
constexpr int DMVR_TAIL = 1640;   // DMVR scratch behind the windows: bilinear 20x20 x2 + their 1-sample-shifted copies (1600), later the
                                  // shifted final windows (2 x 552 luma from 0, 4 x 132 chroma from 1104)
static_assert(4 * 400 <= DMVR_TAIL && 2 * 24 * 23 <= 1104 && 1104 + 4 * 12 * 11 <= DMVR_TAIL, "DMVR scratch");

// Offsets (int16 elements) of a tile's shared arrays, and their total: windows and H-filtered rows of each list, then chroma; boundary DMVR
// tiles first stage two raw 21x21 search windows from 0, and BDOF's 16-byte per-sample records reuse the window area from 0.
struct TileLayout { int w[2], h[2], cw[2][2], chf[2][2], tail, p, total; };
constexpr __host__ __device__ TileLayout tile_layout(int mode, int tw, int th)
{
  TileLayout o{};
  const int lists = mode == 0 ? 1 : 2, cw = tw >> 1, ch = th >> 1;
  int q = 0;
  for (int l = 0; l < lists; l++) { o.w[l] = q; q += (tw + 8) * (th + 7); o.h[l] = q; q += (th + 7) * HS; }
  for (int l = 0; l < lists; l++)
    for (int c = 0; c < 2; c++) { o.cw[l][c] = q; q += (cw + 4) * (ch + 3); o.chf[l][c] = q; q += (ch + 3) * CHS; }
  if (mode == 3 && q < 2 * 441) q = 2 * 441;
  if (mode >= 2 && q < 8 * tw * th) q = 8 * tw * th;
  o.tail = q; if (mode == 3) q += DMVR_TAIL;
  o.p = q; if (mode >= 2) q += 2 * 324;                  // P0/P1 18x18
  o.total = q;
  return o;
}

constexpr __host__ __device__ int mc_size_class(int n) { return n <= 32 ? 0 : n <= 64 ? 1 : n <= 128 ? 2 : 3; }   // as bucket.cu sorts tiles

// Dynamic shared memory of launch class (mode, k), in elements: the largest layout among the tile shapes of 32 << k samples (k = 0 also
// takes 4x4), plus 64 elements of slack
constexpr __host__ __device__ int mc_smem_elems(int mode, int k)
{
  int e = 0;
  for (int tw = 4; tw <= 16; tw *= 2)
    for (int th = 4; th <= 16; th *= 2)
      if (mc_size_class(tw * th) == k && tile_layout(mode, tw, th).total > e) e = tile_layout(mode, tw, th).total;
  return (e + 64) & ~7;
}

// Every legal (MODE, tw, th) carves its arrays inside the allocation of the class bucket.cu sorts it into.  mc_smem_elems is built from
// tile_layout, so this guards the shape enumeration and mc_size_class against each other (e.g. a shape added to one and not the other); the
// kernel and the launch cannot disagree on the carve-up itself, since both take it from tile_layout.
constexpr bool mc_layouts_fit()
{
  for (int mode = 0; mode < 4; mode++)
    for (int tw = 4; tw <= 16; tw *= 2)
      for (int th = 4; th <= 16; th *= 2)
        if ((mode < 2 || tw * th >= 128) && tile_layout(mode, tw, th).total > mc_smem_elems(mode, mc_size_class(tw * th))) return false;
  return true;
}
static_assert(mc_layouts_fit(), "a tile's shared arrays overrun its launch class's dynamic shared memory");

struct McList {               // one list of a translational tile
  const int16_t* ref[3];      // reference planes
  int mvx, mvy;               // MV of the PU (DMVR: the initial MV)
  int fmx, fmy;               // final clipped MV: its fractions select the filters
  int ox, oy, ocx, ocy;       // integer reference position of output sample (0,0), luma / chroma
  Rect rect[2];               // luma / chroma clamp rectangle of the per-sample loads
  bool pad[2];                // DMVR: rect is the padded window of the final MC, so the footprint must be clamped to it
  int wofs, cofs;             // index of the footprint's first sample in each shared window row
};

__device__ __forceinline__ RefView ref_view(const McParams& P, const McList& M, int c) { return {M.ref[c], P.refStride[c ? 1 : 0], M.rect[c ? 1 : 0]}; }

// Stages one list's footprint into shared memory: the luma window (tw+7)x(th+7) from (lx, ly), stride tw+8, and with chroma both chroma
// windows (cw+3)x(ch+3) from (cx, cy), stride cw+4.  An interior window (lfast / cfast) is copied as whole 32-bit words, 16 lanes per luma
// row / 8 lanes per chroma row, asynchronously (the caller waits once); its first sample then sits at index wofs / cofs (0/1) of each shared
// row.  Otherwise each sample is read through M's clamp rectangle, one x clamp per lane.
__device__ __forceinline__ void stage_windows(const McParams& P, McList& M, int tw, int th, int lx, int ly, int cx, int cy, bool lfast, bool cfast,
                                              int16_t* w, int16_t* cb, int16_t* cr)
{
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = max(1, (int)blockDim.x >> 5);
  const int cw = tw >> 1, ch = th >> 1, WS = tw + 8, CS = cw + 4;
  const RefView v = ref_view(P, M, 0);
  M.wofs = lfast ? lx & 1 : 0;
  if (lfast) {
    const int half = lane >> 4, wl = lane & 15, rw = v.stride >> 1;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(v.p + (size_t)ly * v.stride + (lx & ~1)) + (size_t)(warp * 2 + half) * rw + wl;
    uint32_t* dst = reinterpret_cast<uint32_t*>(w) + (warp * 2 + half) * (WS >> 1) + wl;
    if (wl < (WS >> 1))
#pragma unroll 4
      for (int y = warp * 2 + half; y < th + 7; y += nw * 2) { cp_async4(dst, src); src += (size_t)(nw * 2) * rw; dst += nw * 2 * (WS >> 1); }
  } else {
    const int xc = v.cx(lx + lane);
    if (lane < tw + 7)
#pragma unroll 4
      for (int y = warp; y < th + 7; y += nw) w[y * WS + lane] = v.ld(xc, ly + y);
  }
  M.cofs = 0;
  if (!P.chroma) return;
  const RefView vb = ref_view(P, M, 1), vr = ref_view(P, M, 2);
  if (cfast) {
    M.cofs = cx & 1;
    const int sub = lane >> 3, wl = lane & 7, rwc = vb.stride >> 1, npc = (ch + 6) >> 2;   // 4 rows per pass, npc passes per component
    const size_t cbase = (size_t)cy * vb.stride + (cx & ~1);
    for (int q = warp; q < 2 * npc; q += nw) {
      const int c = q >= npc, y = ((c ? q - npc : q) << 2) + sub;
      if (y < ch + 3 && wl < (CS >> 1))
        cp_async4(reinterpret_cast<uint32_t*>(c ? cr : cb) + y * (CS >> 1) + wl, reinterpret_cast<const uint32_t*>((c ? vr.p : vb.p) + cbase) + (size_t)y * rwc + wl);
    }
  } else {
    // both chroma components: lanes 0..15 Cb, 16..31 Cr (cw+3 <= 11)
    const int c = lane >> 4, xl = lane & 15;
    const RefView vc = c ? vr : vb;
    const int xcc = vc.cx(cx + xl);
    int16_t* dc = c ? cr : cb;
    if (xl < cw + 3)
#pragma unroll 4
      for (int y = warp; y < ch + 3; y += nw) dc[y * CS + xl] = vc.ld(xcc, cy + y);
  }
}

// copy of a staged window (w x h samples, stride s) shifted by (dx, dy) and clamped to it: the padded window of DMVR's final MC
__device__ __forceinline__ void shifted_copy(const int16_t* T, int16_t* D, int w, int h, int s, int dx, int dy, int x, int warp, int nw)
{
  const int xs = min(max(x + dx, 0), w - 1);
  if (x < w)
    for (int y = warp; y < h; y += nw) D[y * s + x] = T[min(max(y + dy, 0), h - 1) * s + xs];
}

// ================================================================ DMVR search (xProcessDMVR :1847)
// Stages the search windows, interpolates them bilinearly, sums the 25 SADs, decides the refinement (written to P.dmvrMv), and settles each
// list's final MV and footprint.  Interior tiles copy the 8-tap / 4-tap footprints of the INITIAL motion once (word-wide): the bilinear search
// window (xinitMC :1804, 2 integer samples around the block) is a sub-window of the luma footprint, and the padded window of the final MC
// (xPrefetchPad :1525 / xFinalPaddedMCForDMVR :1731) is that same footprint shifted by the integer part of the refinement and clamped to it;
// then the footprints are staged and the function returns true.  Boundary tiles (footprint touching the picture edge, where MV clipping may
// act) go sample by sample and leave stage A each list's origin and clamp rectangles.
__device__ __forceinline__ bool dmvr_search(const McParams& P, const b200_pu& pu, int tx0, int ty0, int tw, int th, McList (&L)[2], TileSmem& S,
                                            int16_t* smem, int16_t* tail, unsigned* sSad, int* sDec, bool& bio)
{
  const int tid = threadIdx.x, nthr = blockDim.x, warp = tid >> 5, lane = tid & 31, nw = max(1, nthr >> 5);
  const int bx = pu.x + tx0, by = pu.y + ty0, cw = tw >> 1, ch = th >> 1, W = P.W, H = P.H, CWp = W >> 1, CHp = H >> 1;
  const bool chroma = P.chroma;
  int16_t* B0 = tail; int16_t* B1 = tail + 400;            // bilinear buffers 20x20 (stride 20) ...
  int16_t* B0s = tail + 800; int16_t* B1s = tail + 1200;   // ... and copies shifted by one sample, so that every SAD row is word-aligned
  const int BW = tw + 4, BH = th + 4;
  bool fast = P.fastOk;
#pragma unroll
  for (int li = 0; li < 2; li++) {
    const int ix = bx + (L[li].mvx >> 4), iy = by + (L[li].mvy >> 4), icx = (bx >> 1) + (L[li].mvx >> 5), icy = (by >> 1) + (L[li].mvy >> 5);
    fast = fast && ix >= 6 && ix + tw + 8 < W && iy >= 6 && iy + th + 8 < H;
    fast = fast && (!chroma || (icx >= 4 && icx + cw + 5 < CWp && icy >= 3 && icy + ch + 4 < CHp));
  }
  const int16_t* braw[2]; int bstr;                        // raw integer samples of the search window: (BW+1)x(BH+1) per list
  int bxF[2], byF[2];
  if (fast) {
#pragma unroll
    for (int li = 0; li < 2; li++) {
      McList& M = L[li];
      bxF[li] = M.mvx & 15; byF[li] = M.mvy & 15;
      stage_windows(P, M, tw, th, bx + (M.mvx >> 4) - 3, by + (M.mvy >> 4) - 3, (bx >> 1) + (M.mvx >> 5) - 1, (by >> 1) + (M.mvy >> 5) - 1,
                    true, true, S.w[li], S.cw[li][0], S.cw[li][1]);
      braw[li] = S.w[li] + (tw + 8) + M.wofs + 1;
    }
    bstr = tw + 8;
  } else {
    int16_t* R0 = smem;                                    // raw windows, stride 21
    constexpr int NB = 8;
    RefView v[2]; int X0[2], Y0[2];
#pragma unroll
    for (int li = 0; li < 2; li++) {
      int cx = L[li].mvx, cy = L[li].mvy;
      clip_mv(cx, cy, pu.x, pu.y, P);                      // xinitMC :1811: relative to the CU
      const int mx = cx - 32, my = cy - 32;
      v[li] = ref_view(P, L[li], 0);
      bxF[li] = mx & 15; byF[li] = my & 15; X0[li] = v[li].cx(bx + (mx >> 4) + lane); Y0[li] = by + (my >> 4);
      braw[li] = R0 + li * 441;
    }
    bstr = 21;
    if (lane < BW + 1)
      for (int y0 = warp; y0 < BH + 1; y0 += nw * NB) {
        int16_t r[2][NB];
#pragma unroll
        for (int li = 0; li < 2; li++)
#pragma unroll
          for (int k = 0; k < NB; k++) {
            const int y = y0 + k * nw;
            if (y < BH + 1) r[li][k] = v[li].ld(X0[li], Y0[li] + y);
          }
#pragma unroll
        for (int li = 0; li < 2; li++)
#pragma unroll
          for (int k = 0; k < NB; k++) {
            const int y = y0 + k * nw;
            if (y < BH + 1) R0[li * 441 + y * 21 + lane] = r[li][k];
          }
      }
  }
  if (tid < 25) sSad[tid] = 0;
  cp_async_wait_all();
  __syncthreads();
  {
    // bilinear interpolation to 10 bit (filterN2_2D, InterpolationFilter.cpp:1133): one thread per (list, column) walks down the rows
    // and keeps the previous row's horizontal result.  Two-step form; equals the reference's one-step special cases for
    // xF == 0 or yF == 0 at bit depths <= 10.  Coefficients are (16 - frac, frac).
    const int s1 = 4 - (10 - P.bitDepth), o1 = 1 << (s1 - 1);
    for (int i = tid; i < 2 * BW; i += nthr) {
      const int li = i >= BW, x = li ? i - BW : i;
      const int f1 = li ? bxF[1] : bxF[0], f0 = 16 - f1, g1 = li ? byF[1] : byF[0], g0 = 16 - g1;
      const int16_t* r = (li ? braw[1] : braw[0]) + x;
      int16_t* o = (li ? B1 : B0) + x; int16_t* os = (li ? B1s : B0s) + x - 1;
      int prev = (int16_t)((f0 * r[0] + f1 * r[1] + o1) >> s1);
      for (int y = 0; y < BH; y++) {
        r += bstr;
        const int cur = (int16_t)((f0 * r[0] + f1 * r[1] + o1) >> s1);
        const int16_t v = (int16_t)((g0 * prev + g1 * cur + 8) >> 4);
        o[y * 20] = v; if (x) os[y * 20] = v;
        prev = cur;
      }
    }
  }
  __syncthreads();
  {
    // SAD over every second row (RdCost.cpp:113-135): item = (position p, row pair); samples are 10-bit non-negative, so two of them
    // go through one packed max/min/subtract, and the two running halves cannot carry (8 words * 1023 < 2^16)
    const int l2hh = 30 - __clz(th);                       // log2(th / 2)
    for (int it = tid; it < (25 << l2hh); it += nthr) {
      const int p = it >> l2hh, y = (it & ((th >> 1) - 1)) * 2;
      const int u = p % 5 - 2, v = p / 5 - 2, odd = u & 1;
      const uint32_t* a = reinterpret_cast<const uint32_t*>((odd ? B0s : B0) + (2 + v + y) * 20 + 2 + u - odd);
      const uint32_t* b = reinterpret_cast<const uint32_t*>((odd ? B1s : B1) + (2 - v + y) * 20 + 2 - u - odd);
      uint32_t acc = 0;
#pragma unroll 4
      for (int x = 0; x < (tw >> 1); x++) acc += __vmaxs2(a[x], b[x]) - __vmins2(a[x], b[x]);
      atomicAdd(&sSad[p], (acc & 0xffff) + (acc >> 16));
    }
  }
  __syncthreads();
  if (tid == 0) {
    unsigned minCost = sSad[12]; minCost -= minCost >> 2;  // (:1924-1925)
    int dx = 0, dy = 0;
    if (minCost >= (unsigned)(tw * th)) {
      const unsigned c12 = minCost;
      int bi_ = 12;
      for (int i = 0; i < 25; i++) { const unsigned v = i == 12 ? c12 : sSad[i]; if (v < minCost) { minCost = v; bi_ = i; } }   // xBIPMVRefine: raster order, strict <
      const int bu = bi_ % 5 - 2, bv = bi_ / 5 - 2;
      dx = bu * 16; dy = bv * 16;
      if (abs(dx) != 32 && abs(dy) != 32) {                // xDMVRSubPixelErrorSurface / xSubPelErrorSrfc
        auto at = [&](int i) -> unsigned long long { return i == 12 ? c12 : sSad[i]; };
        const unsigned long long s0 = at(bi_), sl = at(bi_ - 1), st = at(bi_ - 5), sr = at(bi_ + 1), sb = at(bi_ + 5);
        { const long long num = (long long)(sl - sr) * 16, den = (long long)(sl + sr - (s0 << 1));
          if (den != 0) dx += (sl != s0 && sr != s0) ? div_for_maxq7(num, den) : (sl == s0 ? -8 : 8); }
        { const long long num = (long long)(st - sb) * 16, den = (long long)(st + sb - (s0 << 1));
          if (den != 0) dy += (st != s0 && sb != s0) ? div_for_maxq7(num, den) : (st == s0 ? -8 : 8); }
      }
    }
    sDec[0] = dx; sDec[1] = dy; sDec[2] = (minCost < (unsigned)(2 * tw * th)) ? 0 : 1;   // bioAppliedSubblk (:1984)
    if (P.dmvrMv) {
      const int num = (ty0 >> 4) * max(1, pu.w >> 4) + (tx0 >> 4);
      P.dmvrMv[(pu.dmvrOff + num) * 2] = dx; P.dmvrMv[(pu.dmvrOff + num) * 2 + 1] = dy;
    }
  }
  __syncthreads();
  bio = (pu.flags & B200_PU_BDOF) && sDec[2];
  const int dmx = sDec[0], dmy = sDec[1];
#pragma unroll
  for (int li = 0; li < 2; li++) {
    McList& M = L[li];
    const int rx = clip3(-(1 << 17), (1 << 17) - 1, li ? M.mvx - dmx : M.mvx + dmx), ry = clip3(-(1 << 17), (1 << 17) - 1, li ? M.mvy - dmy : M.mvy + dmy);
    int cx = rx, cy = ry;
    clip_mv(cx, cy, bx, by, P);                            // cMvClipped, relative to the sub-block (:1749); no-op for interior tiles
    M.fmx = cx; M.fmy = cy;
    if (fast) {
      // shifted + clamped copies of the footprints into the (now free) bilinear scratch
      const int dIx = (rx >> 4) - (M.mvx >> 4), dIy = (ry >> 4) - (M.mvy >> 4);
      if (dIx | dIy) {
        shifted_copy(S.w[li] + M.wofs, tail + li * 552, tw + 7, th + 7, tw + 8, dIx, dIy, lane, warp, nw);
        S.w[li] = tail + li * 552; M.wofs = 0;
      }
      const int dCx = (rx >> 5) - (M.mvx >> 5), dCy = (ry >> 5) - (M.mvy >> 5);
      if (chroma && (dCx | dCy)) {
        const int c = lane >> 4;
        int16_t* D = tail + 1104 + li * 2 * 132;
        shifted_copy((c ? S.cw[li][1] : S.cw[li][0]) + M.cofs, D + c * 132, cw + 3, ch + 3, cw + 4, dCx, dCy, lane & 15, warp, nw);
        S.cw[li][0] = D; S.cw[li][1] = D + 132; M.cofs = 0;
      }
    } else {
#pragma unroll
      for (int k = 0; k < 2; k++) {                        // k = 0 luma, 1 chroma (xFinalPaddedMCForDMVR :1757-1778, xPrefetchPad :1525)
        const int sh = 4 + k, taps = k ? 4 : 8;
        const int dIx = (rx >> sh) - (M.mvx >> sh), dIy = (ry >> sh) - (M.mvy >> sh);
        int X = (bx >> k) + (cx >> sh), Y = (by >> k) + (cy >> sh);
        if (dIx || dIy) {
          int pmx = M.mvx - ((taps / 2 - 1) << sh), pmy = M.mvy - ((taps / 2 - 1) << sh);
          clip_mv(pmx, pmy, bx, by, P);
          const int x0 = (bx >> k) + (pmx >> sh), y0 = (by >> k) + (pmy >> sh), Wk = W >> k, Hk = H >> k;
          M.rect[k] = {clip3(0, Wk - 1, x0), clip3(0, Wk - 1, x0 + (tw >> k) + taps - 2), clip3(0, Hk - 1, y0), clip3(0, Hk - 1, y0 + (th >> k) + taps - 2)};
          M.pad[k] = true;
          X = x0 + (taps / 2 - 1) + dIx; Y = y0 + (taps / 2 - 1) + dIy;
        }
        if (k == 0) { M.ox = X; M.oy = Y; } else { M.ocx = X; M.ocy = Y; }
      }
    }
  }
  return fast;
}

// OPT: luma outputs per thread (1: blockDim = tw*th; 4: blockDim = tw*th/4, each thread filters 4 adjacent samples so that 11 loads feed 32 MACs)
template <int MODE, int OPT>
__device__ __forceinline__ void mc_tile(const McParams& P, const uint32_t tile, int16_t* smem, unsigned* sSad, int* sDec, int (*sVxy)[2])
{
  const int tid = threadIdx.x, nthr = blockDim.x;
  const b200_pu& pu = P.pus[tile >> 6];
  const int puW = pu.w, puH = pu.h, puX = pu.x, puY = pu.y, flags = pu.flags;
  const int tx0 = (tile & 7) * 16, ty0 = ((tile >> 3) & 7) * 16;
  const int tw = min(16, puW - tx0), th = min(16, puH - ty0);
  const int l2w = 31 - __clz(tw);
  const int bx = puX + tx0, by = puY + ty0;
  const int bd = P.bitDepth, pmax = (1 << bd) - 1, hr = max(2, 14 - bd), sh1 = 6 - hr;
  constexpr bool BI = MODE != 0;
  const bool altHpel = flags & B200_PU_ALTHPEL;
  const bool is4x4 = puW == 4 && puH == 4;
  const int l0 = BI ? 0 : (pu.refSlot[0] >= 0 ? 0 : 1);     // first (or only) list
  constexpr int NL = BI ? 2 : 1;
  const int cw = tw >> 1, ch = th >> 1, l2cw = l2w - 1;
  const int chroma = P.chroma;
  const b200_wp* we = (MODE <= 1 && P.wp && pu.wpIdx) ? P.wp + pu.wpIdx - 1 : nullptr;   // explicit weights (never with BDOF / DMVR)
  const bool geo = MODE == 1 && (flags & B200_PU_GEO);      // geometric partitioning: the two 'lists' are the two partitions' uni-predictions
  const int gl2w = 31 - __clz(puW), gl2h = 31 - __clz(puH);
  const int WS = tw + 8, CS = cw + 4;                        // window strides: even, so a row is a run of 32-bit words

  const TileLayout Lo = tile_layout(MODE, tw, th);
  TileSmem S;
#pragma unroll
  for (int l = 0; l < NL; l++) {
    S.w[l] = smem + Lo.w[l]; S.h[l] = smem + Lo.h[l];
#pragma unroll
    for (int c = 0; c < 2; c++) { S.cw[l][c] = smem + Lo.cw[l][c]; S.chf[l][c] = smem + Lo.chf[l][c]; }
  }
  S.p[0] = smem + Lo.p; S.p[1] = S.p[0] + 324;

  // ---- motion per list ----
  const int W = P.W, H = P.H, CWp = W >> 1, CHp = H >> 1;
  McList L[NL];
#pragma unroll
  for (int li = 0; li < NL; li++) {
    const int l = BI ? li : l0;
    const int slot = pu.refSlot[l];
#pragma unroll
    for (int c = 0; c < 3; c++) L[li].ref[c] = P.refs[slot * 3 + c];
    L[li].mvx = pu.mv[l][0]; L[li].mvy = pu.mv[l][1];
    L[li].rect[0] = {0, W - 1, 0, H - 1}; L[li].rect[1] = {0, CWp - 1, 0, CHp - 1}; L[li].pad[0] = L[li].pad[1] = false;
  }
  bool bio = MODE == 2, staged = false;
  if constexpr (MODE == 3) staged = dmvr_search(P, pu, tx0, ty0, tw, th, L, S, smem, smem + Lo.tail, sSad, sDec, bio);
  else {
#pragma unroll
    for (int li = 0; li < NL; li++) {
      int cx = L[li].mvx, cy = L[li].mvy;
      clip_mv(cx, cy, puX, puY, P);                          // relative to the CU (xPredInterUni :651)
      L[li].fmx = cx; L[li].fmy = cy;
      L[li].ox = bx + (cx >> 4); L[li].oy = by + (cy >> 4); L[li].ocx = (bx >> 1) + (cx >> 5); L[li].ocy = (by >> 1) + (cy >> 5);
    }
  }

  // ================================================================ stage A: windows (luma 8-tap footprint, chroma 4-tap footprint)
  // Interior tiles (the footprint lies inside the picture and no DMVR window clamp applies) copy whole words; boundary tiles load each sample
  // through the clamp rectangle (= the reference's border extension / padded DMVR window).
  if (!staged) {
#pragma unroll
    for (int li = 0; li < NL; li++) {
      McList& M = L[li];
      const bool lfast = P.fastOk && !M.pad[0] && M.ox >= 4 && M.ox + tw + 4 < W && M.oy >= 3 && M.oy + th + 3 < H;
      const bool cfast = P.fastOk && !M.pad[1] && M.ocx >= 2 && M.ocx + cw + 2 < CWp && M.ocy >= 1 && M.ocy + ch + 1 < CHp;
      stage_windows(P, M, tw, th, M.ox - 3, M.oy - 3, M.ocx - 1, M.ocy - 1, lfast, cfast, S.w[li], S.cw[li][0], S.cw[li][1]);
    }
  }
  cp_async_wait_all();
  __syncthreads();

  // ================================================================ stage B: horizontal filters
#pragma unroll
  for (int li = 0; li < NL; li++) {
    int f[8];
    load_taps8(luma_taps(L[li].fmx & 15, is4x4, altHpel), f);  // row 0 of the tables is {0,0,0,64,0,0,0,0}: full-pel is the same formula
    const int16_t* sw = S.w[li] + L[li].wofs;
    if (OPT == 1) {
      for (int i = tid; i < (th + 7) << l2w; i += nthr) {
        const int y = i >> l2w, x = i & (tw - 1);
        const int16_t* s = sw + y * WS + x;
        int a = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) a += f[k] * s[k];
        S.h[li][y * HS + x] = (int16_t)((a - (IFO << sh1)) >> sh1);
      }
    } else {
      const int l2g = l2w - 2;                               // groups of 4 outputs per row
      for (int i = tid; i < (th + 7) << l2g; i += nthr) {
        const int y = i >> l2g, x = (i & ((tw >> 2) - 1)) << 2;
        const int16_t* s = sw + y * WS + x;
        int v[11];
#pragma unroll
        for (int k = 0; k < 11; k++) v[k] = s[k];
        int16_t* o = S.h[li] + y * HS + x;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          int a = 0;
#pragma unroll
          for (int k = 0; k < 8; k++) a += f[k] * v[j + k];
          o[j] = (int16_t)((a - (IFO << sh1)) >> sh1);
        }
      }
    }
    if (chroma) {
      const int8_t* t = kIfChroma + (L[li].fmx & 31) * 4;
      const int c0 = t[0], c1 = t[1], c2 = t[2], c3 = t[3];
      for (int i = tid; i < 2 * ((ch + 3) << l2cw); i += nthr) {
        const int c = i >= ((ch + 3) << l2cw), j = c ? i - ((ch + 3) << l2cw) : i;
        const int y = j >> l2cw, x = j & (cw - 1);
        const int16_t* s = (c ? S.cw[li][1] : S.cw[li][0]) + L[li].cofs + y * CS + x;
        (c ? S.chf[li][1] : S.chf[li][0])[y * CHS + x] = (int16_t)((c0 * s[0] + c1 * s[1] + c2 * s[2] + c3 * s[3] - (IFO << sh1)) >> sh1);
      }
    }
  }
  __syncthreads();

  // ================================================================ stage C: vertical filters + combine
  // thread -> samples (x, y0 .. y0+OPT-1); with BDOF the same thread keeps its samples' terms in registers until the final combine
  const int sx = tid & (tw - 1), sy = (tid >> l2w) * OPT;
  const int w1 = MODE == 1 ? pu.bcwW1 : 4;
  {
    int pr[NL][OPT];
#pragma unroll
    for (int li = 0; li < NL; li++) {
      int f[8];
      load_taps8(luma_taps(L[li].fmy & 15, is4x4, altHpel), f);
      const int16_t* s = S.h[li] + sy * HS + sx;
      int v[7 + OPT];
#pragma unroll
      for (int k = 0; k < 7 + OPT; k++) v[k] = s[k * HS];
#pragma unroll
      for (int j = 0; j < OPT; j++) {
        int a = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) a += f[k] * v[j + k];
        pr[li][j] = a;
      }
    }
#pragma unroll
    for (int j = 0; j < OPT; j++) {
      if (OPT == 1 && sy >= th) break;                       // a 4x4 tile runs in the 32-thread launch of its class: threads 16..31 have no sample
      const int p0 = BI ? (int16_t)(pr[0][j] >> 6) : pr[0][j], p1 = (int16_t)(pr[NL - 1][j] >> 6);
      if (bio) { S.p[0][(sy + j + 1) * 18 + sx + 1] = (int16_t)p0; S.p[1][(sy + j + 1) * 18 + sx + 1] = (int16_t)p1; continue; }
      const int gw = geo ? geo_weight(pu.bcwW1, gl2w, gl2h, tx0 + sx, ty0 + sy + j, 0) : -1;
      P.dst[0][(size_t)(by + sy + j) * P.dstStride[0] + bx + sx] = (int16_t)mc_sample(P, 0, BI ? MC_BI14 : MC_UNI_SUM, we, gw, w1, p0, p1, hr, pmax);
    }
  }
  if (chroma) {
    for (int i = tid; i < 2 * (ch << l2cw); i += nthr) {
      const int c = i >= (ch << l2cw), j = c ? i - (ch << l2cw) : i;
      const int y = j >> l2cw, x = j & (cw - 1);
      int pr[NL];
#pragma unroll
      for (int li = 0; li < NL; li++) {
        const int8_t* t = kIfChroma + (L[li].fmy & 31) * 4;
        const int16_t* s = (c ? S.chf[li][1] : S.chf[li][0]) + y * CHS + x;
        pr[li] = t[0] * s[0] + t[1] * s[CHS] + t[2] * s[2 * CHS] + t[3] * s[3 * CHS];
      }
      const int gw = geo ? geo_weight(pu.bcwW1, gl2w, gl2h, (tx0 >> 1) + x, (ty0 >> 1) + y, 1) : -1;
      (c ? P.dst[2] : P.dst[1])[(size_t)((by >> 1) + y) * (c ? P.dstStride[2] : P.dstStride[1]) + (bx >> 1) + x] =
          (int16_t)mc_sample(P, 1 + c, BI ? MC_BI14 : MC_UNI_SUM, we, gw, w1, BI ? (int16_t)(pr[0] >> 6) : pr[0], (int16_t)(pr[NL - 1] >> 6), hr, pmax);
    }
  }

  // ================================================================ BDOF (applyBiOptFlow :1290)
  if (MODE >= 2) {
    if (!bio) return;                                        // CTA-uniform
    // ring of integer reference samples around the block (xPredInterBlk :847-885); the windows already hold them
    for (int i = tid; i < 4 * (tw + th + 2); i += nthr) {
      const int li = i >= 2 * (tw + th + 2), j = li ? i - 2 * (tw + th + 2) : i;
      int x, y;
      if (j < tw + 2) { x = j; y = 0; } else if (j < 2 * (tw + 2)) { x = j - (tw + 2); y = th + 1; }
      else if (j < 2 * (tw + 2) + th) { x = 0; y = j - 2 * (tw + 2) + 1; } else { x = tw + 1; y = j - 2 * (tw + 2) - th + 1; }
      const int mxl = li ? L[NL - 1].fmx : L[0].fmx, myl = li ? L[NL - 1].fmy : L[0].fmy;
      const int xo = (mxl & 15) < 8 ? 1 : 0, yo = (myl & 15) < 8 ? 1 : 0;
      const int16_t* wl = li ? S.w[NL - 1] + L[NL - 1].wofs : S.w[0] + L[0].wofs;
      const int v = wl[(y - yo + 3) * WS + (x - xo + 3)];
      (li ? S.p[1] : S.p[0])[y * 18 + x] = (int16_t)((int16_t)(v << hr) - IFO);
    }
    __syncthreads();
    // per sample: gradients of both lists (gradFilterCore<true> :212) folded into the five summands of calcBIOSums (:134), one 16-byte
    // record per sample; the padded border of the reference (PaddBIOCore :269, replication of the outermost samples) becomes a clamp of
    // the record index when the 6x6 windows are summed.  The terms of the final combine stay in this thread's registers.
    uint4* Q = reinterpret_cast<uint4*>(smem);
    int dgx[OPT], dgy[OPT], psum[OPT];
    {
      int q0[OPT + 2], q1[OPT + 2];                          // column sx, rows sy-1 .. sy+OPT (>> 6)
#pragma unroll
      for (int r = 0; r < OPT + 2; r++) { q0[r] = S.p[0][(sy + r) * 18 + sx + 1] >> 6; q1[r] = S.p[1][(sy + r) * 18 + sx + 1] >> 6; }
#pragma unroll
      for (int j = 0; j < OPT; j++) {
        const int i = (sy + j + 1) * 18 + sx + 1;
        const int p0 = S.p[0][i], p1 = S.p[1][i];
        const int g0x = (S.p[0][i + 1] >> 6) - (S.p[0][i - 1] >> 6), g1x = (S.p[1][i + 1] >> 6) - (S.p[1][i - 1] >> 6);
        const int g0y = q0[j + 2] - q0[j], g1y = q1[j + 2] - q1[j];
        const int tX = (g0x + g1x) >> 1, tY = (g0y + g1y) >> 1, dI = (p1 >> 4) - (p0 >> 4);
        uint4 rec;
        rec.x = (unsigned)abs(tX) | ((unsigned)abs(tY) << 16);
        rec.y = (unsigned)(tX < 0 ? -dI : (tX == 0 ? 0 : dI));
        rec.z = (unsigned)(tY < 0 ? -dI : (tY == 0 ? 0 : dI));
        rec.w = (unsigned)(tY < 0 ? -tX : (tY == 0 ? 0 : tX));
        Q[((sy + j) << l2w) + sx] = rec;
        dgx[j] = g0x - g1x; dgy[j] = g0y - g1y; psum[j] = p0 + p1;
      }
    }
    __syncthreads();
    const int nBlk = (tw >> 2) * (th >> 2), l2bw = l2w - 2;
    // 4 lanes per 4x4 block: lane part p sums window rows p and p+4 (rows 4,5 only for p<2); quad shuffle reduce; lane 0 derives (vx,vy)
    for (int it = tid; it < ((nBlk * 4 + 31) & ~31); it += nthr) {
      const int blk = it >> 2, part = it & 3;
      unsigned sA = 0; int sDX = 0, sDY = 0, sS = 0;
      if (blk < nBlk) {
        const int bxx = (blk & ((tw >> 2) - 1)) << 2, byy = (blk >> l2bw) << 2;
#pragma unroll
        for (int rr = 0; rr < 2; rr++) {
          const int yy = part + 4 * rr;
          if (yy < 6) {
            const uint4* row = Q + (min(max(byy + yy - 1, 0), th - 1) << l2w);
#pragma unroll
            for (int xx = 0; xx < 6; xx++) {
              const uint4 r = row[min(max(bxx + xx - 1, 0), tw - 1)];
              sA += r.x; sDX += (int)r.y; sDY += (int)r.z; sS += (int)r.w;
            }
          }
        }
      }
#pragma unroll
      for (int m = 1; m < 4; m <<= 1) {
        sA += __shfl_xor_sync(0xffffffffu, sA, m);
        sDX += __shfl_xor_sync(0xffffffffu, sDX, m); sDY += __shfl_xor_sync(0xffffffffu, sDY, m);
        sS  += __shfl_xor_sync(0xffffffffu, sS, m);
      }
      if (part == 0 && blk < nBlk) {
        const int sAX = sA & 0xffff, sAY = sA >> 16;         // 36 * 256 < 2^16: the packed halves cannot carry
        int vx = sAX == 0 ? 0 : shift_msb(sDX * 4, sAX);
        vx = clip3(-15, 15, vx);
        const int mainG = sS >> 12, secG = sS & 4095;
        int tmp = vx * mainG;
        tmp = ((tmp * (1 << 12)) + vx * secG) >> 1;
        int vy = sAY == 0 ? 0 : shift_msb(sDY * 4 - tmp, sAY);
        vy = clip3(-15, 15, vy);
        sVxy[blk][0] = vx; sVxy[blk][1] = vy;
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < OPT; j++) {                          // addBIOAvg4 (:109)
      const int y = sy + j, blk = ((y >> 2) << l2bw) + (sx >> 2);
      const int b = sVxy[blk][0] * dgx[j] + sVxy[blk][1] * dgy[j];
      const int shiftNum = 15 - bd, offset = (1 << (shiftNum - 1)) + 2 * IFO;
      P.dst[0][(size_t)(by + y) * P.dstStride[0] + bx + sx] = (int16_t)luma_out(P, clip3(0, pmax, (int)(int16_t)((psum[j] + b + offset) >> shiftNum)), pmax);
    }
  }
}

// One CTA per entry of one tile list (bucket.cu); the host sizes the grid from the list length it reads back after bucketing, and the
// hardware scheduler balances the lists of all streams.
template <int MODE, int OPT>
__global__ void __launch_bounds__(64, MODE >= 2 ? 12 : 16) mc_kernel(const McParams P, const int list)
{
  extern __shared__ __align__(128) int16_t smem[];
  __shared__ unsigned sSad[25];
  __shared__ int sDec[3];
  __shared__ int sVxy[16][2];
  if ((int)blockIdx.x >= P.meta[LM_CNT + list]) return;
  mc_tile<MODE, OPT>(P, P.tiles[P.meta[LM_OFF + list] + blockIdx.x], smem, sSad, sDec, sVxy);
}

// ------------------------------------------------------------------------------------------------ affine tiles (xPredAffineBlk :934)
// the sub-block MVs (round_affine, spread_over_limit, aff_model, aff_sub_mv): affine_mv.cuh

__device__ __forceinline__ void mc_affine_tile(const McParams& P, const uint32_t tile)
{
  __shared__ int16_t sHf[2][16][9 * 4];     // per sub-block: 9 rows x 4 cols after horizontal filter
  __shared__ int16_t sE[2][16][36];         // PROF 6x6 buffers
  __shared__ int16_t sP[2][3][256];         // 14-bit predictions (luma 16x16, chroma 8x8 each)
  __shared__ int16_t sCH[2][2][4][7 * 4];   // chroma: [list][comp][sub-block] 7 rows x 4 cols

  const int tid = threadIdx.x;
  const b200_pu& pu = P.pus[tile >> 6];                      // read in place: per-list fields are indexed at run time, a private copy would live in local memory
  const int tx0 = (tile & 7) * 16, ty0 = ((tile >> 3) & 7) * 16;
  const int tw = min(16, pu.w - tx0), th = min(16, pu.h - ty0);
  const int bx = pu.x + tx0, by = pu.y + ty0;
  const int bd = P.bitDepth, pmax = (1 << bd) - 1, hr = max(2, 14 - bd), sh1 = 6 - hr;
  const bool bi = pu.refSlot[0] >= 0 && pu.refSlot[1] >= 0;
  const b200_wp* we = (P.wp && pu.wpIdx) ? P.wp + pu.wpIdx - 1 : nullptr;
  const int nList = bi ? 2 : 1, l0 = pu.refSlot[0] >= 0 ? 0 : 1;
  const int hMin = (-P.ctuSize - 8 - pu.x + 1) * 16, hMax = (P.W + 8 - pu.x - 1) * 16;
  const int vMin = (-P.ctuSize - 8 - pu.y + 1) * 16, vMax = (P.H + 8 - pu.y - 1) * 16;


  // ---- luma: sub-block sb = tid>>4 (4x4 grid in the tile), lane k = tid&15 ----
  const int sb = tid >> 4, k = tid & 15;
  const int sbx = (sb & 3) * 4, sby = (sb >> 2) * 4;
  const bool sbValid = sbx < tw && sby < th;
  for (int li = 0; li < nList; li++) {
    const int l = bi ? li : l0;
    AffModel Ml; aff_model(pu, l, Ml);                       // per list, in registers
    const RefView Rl = {P.refs[pu.refSlot[l] * 3], P.refStride[0], {0, P.W - 1, 0, P.H - 1}};
    int mx = 0, my = 0;
    if (sbValid) { aff_sub_mv(Ml, pu, (tx0 + sbx) >> 2, (ty0 + sby) >> 2, mx, my); mx = clip3(hMin, hMax, mx); my = clip3(vMin, vMax, my); }
    const int xF = mx & 15, yF = my & 15, X0 = bx + sbx + (mx >> 4), Y0 = by + sby + (my >> 4);
    if (sbValid) {
      const int8_t* fh = kIfLuma4x4 + xF * 8;
      for (int j = k; j < 36; j += 16) {                      // 9 rows (y-2..y+6: 6-tap taps 1..6 of the 8-tap array) x 4 cols
        const int y = j >> 2, x = j & 3;
        int s = 0;
        if (xF == 0) s = 64 * Rl.at(X0 + x, Y0 + y - 2);
        else {
#pragma unroll
          for (int t = 1; t < 7; t++) s += fh[t] * Rl.at(X0 + x + t - 3, Y0 + y - 2);
        }
        sHf[l][sb][j] = (int16_t)((s - (IFO << sh1)) >> sh1);
      }
      if (Ml.prof) {                                       // ring of the 6x6 PROF buffer from integer samples (:1233-1262)
        const int rx = X0 + (xF >> 3) - 1, ry = Y0 + (yF >> 3) - 1;
        for (int j = k; j < 36; j += 16) {
          const int y = j / 6, x = j - y * 6;
          if (x > 0 && x < 5 && y > 0 && y < 5) continue;
          sE[l][sb][j] = (int16_t)((int16_t)(Rl.at(rx + x, ry + y) << hr) - IFO);
        }
      }
    }
    __syncwarp();
    if (sbValid) {
      const int y = k >> 2, x = k & 3;
      const int8_t* fv = kIfLuma4x4 + yF * 8;
      int s = 0;
      if (yF == 0) s = 64 * sHf[l][sb][(y + 2) * 4 + x];
      else {
#pragma unroll
        for (int t = 1; t < 7; t++) s += fv[t] * sHf[l][sb][(y + t - 1) * 4 + x];
      }
      if (Ml.prof) sE[l][sb][(y + 1) * 6 + x + 1] = (int16_t)(s >> 6);
      else if (bi)   sP[l][0][(sby + y) * 16 + sbx + x] = (int16_t)(s >> 6);
      else P.dst[0][(size_t)(by + sby + y) * P.dstStride[0] + bx + sbx + x] = (int16_t)mc_sample(P, 0, MC_UNI_SUM, we, -1, 4, s, 0, hr, pmax);
    }
    __syncwarp();
    if (sbValid && Ml.prof) {                              // gradFilterCore<false> :212 + applyPROFCore :61
      const int y = k >> 2, x = k & 3, c = (y + 1) * 6 + x + 1;
      const int16_t* E = sE[l][sb];
      const int gX = (E[c + 1] >> 6) - (E[c - 1] >> 6), gY = (E[c + 6] >> 6) - (E[c - 6] >> 6);
      // dMv of sample (x,y) inside the 4x4 (:1043-1090): linear in x,y, then rounded by 8 and clipped to +-31
      const int qHX = Ml.dHX * 4, qHY = Ml.dHY * 4, qVX = Ml.dVX * 4, qVY = Ml.dVY * 4;
      int dh = ((Ml.dHX + Ml.dVX) * 2) - ((qHX + qVX) * 2) + x * qHX + y * qVX;
      int dv = ((Ml.dHY + Ml.dVY) * 2) - ((qHY + qVY) * 2) + x * qHY + y * qVY;
      round_affine(dh, dv, 8);
      dh = clip3(-31, 31, dh); dv = clip3(-31, 31, dv);
      const int lim = 1 << max(bd + 1, 13);
      const int dI = clip3(-lim, lim - 1, dh * gX + dv * gY);
      int v = (int16_t)(E[c] + dI);
      if (bi) sP[l][0][(sby + y) * 16 + sbx + x] = (int16_t)v;
      else P.dst[0][(size_t)(by + sby + y) * P.dstStride[0] + bx + sbx + x] = (int16_t)mc_sample(P, 0, MC_UNI14, we, -1, 4, v, 0, hr, pmax);
    }
  }

  // ---- chroma 4:2:0: 4x4 chroma sub-blocks (= 8x8 luma), MV = rounded mean of the TL and BR luma sub-block MVs (:1135-1151) ----
  if (P.chroma) {
    // jobs: (list, comp, chroma sub-block 0..3): 16 threads each -> nList*2*4*16 = 128/256 threads
    const int job = tid >> 4;
    const int li = job >> 3, c = 1 + ((job >> 2) & 1), cs = job & 3;
    const int l = bi ? li : l0;
    const int csx = (cs & 1) * 4, csy = (cs >> 1) * 4;       // chroma offset inside the 8x8 chroma tile
    const bool valid = li < nList && csx < (tw >> 1) && csy < (th >> 1);
    int mx = 0, my = 0;
    RefView Rc = {nullptr, P.refStride[1], {0, (P.W >> 1) - 1, 0, (P.H >> 1) - 1}};
    if (valid) {
      AffModel Ml; aff_model(pu, l, Ml);
      Rc.p = P.refs[pu.refSlot[l] * 3 + c]; Rc.stride = c == 1 ? P.refStride[1] : P.refStride[2];
      int ax, ay, bxm, bym;
      const int i0 = (tx0 >> 2) + (csx >> 1), j0 = (ty0 >> 2) + (csy >> 1);
      aff_sub_mv(Ml, pu, i0, j0, ax, ay); aff_sub_mv(Ml, pu, i0 + 1, j0 + 1, bxm, bym);
      mx = ax + bxm; my = ay + bym;
      round_affine(mx, my, 1);
      mx = clip3(hMin, hMax, mx); my = clip3(vMin, vMax, my);
    }
    const int xF = mx & 31, yF = my & 31, X0 = (bx >> 1) + csx + (mx >> 5), Y0 = (by >> 1) + csy + (my >> 5);
    if (valid) {
      const int8_t* fh = kIfChroma + xF * 4;
      for (int j = k; j < 28; j += 16) {
        const int y = j >> 2, x = j & 3;
        int s = 0;
#pragma unroll
        for (int t = 0; t < 4; t++) s += fh[t] * Rc.at(X0 + x + t - 1, Y0 + y - 1);
        sCH[li][c - 1][cs][j] = (int16_t)((s - (IFO << sh1)) >> sh1);
      }
    }
    __syncwarp();
    if (valid) {
      const int y = k >> 2, x = k & 3;
      const int8_t* fv = kIfChroma + yF * 4;
      int s = 0;
#pragma unroll
      for (int t = 0; t < 4; t++) s += fv[t] * sCH[li][c - 1][cs][(y + t) * 4 + x];
      if (bi) sP[l][c][(csy + y) * 8 + csx + x] = (int16_t)(s >> 6);
      else P.dst[c][(size_t)((by >> 1) + csy + y) * P.dstStride[c] + (bx >> 1) + csx + x] = (int16_t)mc_sample(P, c, MC_UNI_SUM, we, -1, 4, s, 0, hr, pmax);
    }
  }
  if (!bi) return;
  __syncthreads();
  {
    const int y = tid >> 4, x = tid & 15;
    if (x < tw && y < th) P.dst[0][(size_t)(by + y) * P.dstStride[0] + bx + x] = (int16_t)mc_sample(P, 0, MC_BI14, we, -1, pu.bcwW1, sP[0][0][y * 16 + x], sP[1][0][y * 16 + x], hr, pmax);
    if (P.chroma && tid < 128) {
      const int c = 1 + (tid >> 6), j = tid & 63, yy = j >> 3, xx = j & 7;
      if (xx < (tw >> 1) && yy < (th >> 1))
        P.dst[c][(size_t)((by >> 1) + yy) * P.dstStride[c] + (bx >> 1) + xx] = (int16_t)mc_sample(P, c, MC_BI14, we, -1, pu.bcwW1, sP[0][c][yy * 8 + xx], sP[1][c][yy * 8 + xx], hr, pmax);
    }
  }
}

__global__ void __launch_bounds__(256) mc_affine_kernel(const McParams P)
{
  if ((int)blockIdx.x >= P.meta[LM_CNT + 16]) return;
  mc_affine_tile(P, P.tiles[P.meta[LM_OFF + 16] + blockIdx.x]);
}

// [MODE][k >= 2]: 128- / 256-sample tiles filter 4 luma outputs per thread; BDOF / DMVR tiles have at least 128 samples (bucket.cu rejects others)
static void (*const kMcKernels[4][2])(const McParams, int) = {
  {mc_kernel<0, 1>, mc_kernel<0, 4>}, {mc_kernel<1, 1>, mc_kernel<1, 4>}, {nullptr, mc_kernel<2, 4>}, {nullptr, mc_kernel<3, 4>}};

int launch_mc(const McLaunch& L, StreamSet& ss, KHook* hook)
{
  McParams P;
  for (int c = 0; c < 3; c++) { P.dst[c] = L.dst.p[c]; P.dstStride[c] = L.dst.stride[c]; P.refStride[c] = L.refStride[c]; }
  for (int i = 0; i < B200_MAX_SLOTS * 3; i++) P.refs[i] = L.refs[i];
  P.fastOk = !(L.refStride[0] & 1) && !(L.refStride[1] & 1) && !(L.refStride[2] & 1);
  P.W = L.geom.width; P.H = L.geom.height; P.bitDepth = L.geom.bitDepth; P.ctuSize = L.geom.ctuSize; P.chroma = L.geom.chromaFormat == 1;
  P.pus = L.pus; P.dmvrMv = L.dmvrMv; P.tiles = L.tiles; P.meta = L.meta;
  P.wp = L.wp;
  P.lmcs = L.lmcs; P.lmcsLog2 = 0; { int o = (1 << L.geom.bitDepth) / 16; while ((1 << (P.lmcsLog2 + 1)) <= o) P.lmcsLog2++; }
  int launched = 0;
  hook_begin(hook, B200_KF_MC_TILE, ss.main);
  for (int m = 3; m >= 0; m--) for (int k = 3; k >= 0; k--) {      // heaviest lists first (DMVR 16x16 ... uni 8x4)
    const int nsamp = 32 << k, list = m * 4 + k, grid = L.cnt[list];
    if (!grid || (m >= 2 && k < 2)) continue;
    cudaStream_t s = ss.pick(launched++);
    kMcKernels[m][k >= 2]<<<grid, k >= 2 ? nsamp >> 2 : nsamp, (size_t)mc_smem_elems(m, k) * 2, s>>>(P, list);
    hook_count(hook);
    B200_CUDA(cudaGetLastError());
  }
  if (L.cnt[16]) { cudaStream_t s = ss.pick(launched++); mc_affine_kernel<<<L.cnt[16], 256, 0, s>>>(P); hook_count(hook); B200_CUDA(cudaGetLastError()); }
  ss.join();
  hook_end(hook, B200_KF_MC_TILE, ss.main);      // with forked streams the affine tiles are inside the same interval
  return 0;
}

}  // namespace b200
