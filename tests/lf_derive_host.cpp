// lf_derive_host.cpp — the device edge derivation (vvdec_b200/csrc/lf_derive.cuh) compiled for the host, for tests/test_lf_derive_cpu.py, which builds it with
// the host C++ compiler into a temporary directory.  lf_derive_host() takes the arguments of b200_lf_derive and runs lf_derive_serial, the order the device keeps.
#include <vector>
#include "../vvdec_b200/csrc/vvc_tables.h"
#include "../vvdec_b200/csrc/lf_derive.cuh"

extern "C" int lf_derive_host(const b200_geom* g, const b200_lf_cu* cus, size_t numCus, const b200_lf_tu* tus, size_t numTus, const uint32_t* ctuCus,
                              const b200_pu* pus, size_t numPus, const b200_lf_slice* slices, const uint8_t* sliceB, int numSlices, b200_lf_param* lfV, b200_lf_param* lfH)
{
  (void)numTus; (void)numSlices;
  const size_t n4 = (size_t)(g->width >> 2) * (g->height >> 2);
  const int nCtu = ((g->width + g->ctuSize - 1) / g->ctuSize) * ((g->height + g->ctuSize - 1) / g->ctuSize);
  std::vector<uint32_t> m0(n4), m1(n4); std::vector<b200::LfMi> mi(n4);
  b200::LfDerive G{};
  G.W4 = g->width >> 2; G.H4 = g->height >> 2; G.ctuSize = g->ctuSize; G.chroma = g->chromaFormat; G.qpBdOffset2 = 12 * (g->bitDepth - 8);
  G.cus = cus; G.tus = tus; G.pus = pus; G.numPus = numPus; G.cuMap[0] = m0.data(); G.cuMap[1] = m1.data(); G.mi = mi.data();
  G.slices = slices; G.sliceB = sliceB; G.grid[0] = lfV; G.grid[1] = lfH;
  uint32_t* const maps[2] = {m0.data(), m1.data()};
  b200::lf_derive_serial(G, maps, numCus, ctuCus, nCtu, kGeoParams);
  return 0;
}
