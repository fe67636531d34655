// emu_closure_narrow.cc -- drives closure_meet over a 16-bit closure index (spicedb-kubeapi-proxy_b200/csrc/kernels.cuh,
// the two-level meet that deals 32-byte sectors out to the warp) under the CPU SIMT emulator (cuda_emu.h), with an index
// built by the caller. TEST INFRASTRUCTURE ONLY (built by tests/test_closure_narrow_emulation.py into its own .so;
// never part of libzgpu.so).
#define ZG_EMULATE 1
#include "cuda_emu.h"

#include "../../spicedb-kubeapi-proxy_b200/csrc/kernels.cuh"

using namespace zg;

namespace {

struct Args {
  const uint32_t* col;    // the ranges' children
  const uint32_t* crow;   // closure index: nsubj + 1 row offsets
  const uint16_t* ccol;   //   and its 16-bit entries (padded to whole 32-byte sectors)
  uint32_t nsubj;
  const uint32_t* lanes;  // per lane: want, lo, hi, subject, job slot
  uint32_t* hits;         // per warp: job slots answered
  unsigned long long* bytes;  // per lane: the COUNT variant's bytes
};

// One warp per block. A lane's row is looked up as visit() does; lanes that do not want the meet stand for those
// whose step has no index or that have nothing to meet.
void meet_kernel(const Args& a) {
  ZG_DYNAMIC_SMEM(smem);
  const uint32_t lane = threadIdx.x & 31, warp = blockIdx.x;
  const uint32_t* l = a.lanes + (static_cast<size_t>(warp) * 32 + lane) * 5;
  bool want = l[0] != 0;
  const uint32_t lo = l[1], hi = l[2], sid = l[3], jslot = l[4];
  uint32_t rb = 0, re = 0;
  unsigned long long nb = 0;
  if (want && sid < a.nsubj) {
    rb = __ldg(a.crow + sid);
    re = __ldg(a.crow + sid + 1);
    nb += 8;
  }
  want = want && re > rb;
  unsigned long long cb = 0;
  const unsigned h = closure_meet<true>(a.col, a.ccol, reinterpret_cast<unsigned long long*>(smem), lane, want, lo, hi, rb,
                                        re, jslot, &cb);
  if (lane == 0) a.hits[warp] = h;
  a.bytes[static_cast<size_t>(warp) * 32 + lane] = nb + cb;
}

}  // namespace

extern "C" int emu_closure_meet_narrow(const uint32_t* col, const uint32_t* crow, const uint16_t* ccol, uint32_t nsubj,
                                       const uint32_t* lanes, uint32_t n_warps, uint32_t* hits, unsigned long long* bytes) {
  const Args a{col, crow, ccol, nsubj, lanes, hits, bytes};
  zg_emu::launch(meet_kernel, a, n_warps, 32, kMeetWords * sizeof(uint32_t));
  return 0;
}
