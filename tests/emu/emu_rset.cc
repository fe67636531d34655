// emu_rset.cc -- the check kernel over closure indexes, with the slots' SF_NO_RSET flags on or off, under the CPU SIMT
// emulator (cuda_emu.h): emu_main.cc's engine, plus a host build of the 16-bit closure index of every two-level pair
// (what build.cu gpu_build_closure builds on the device) and schema.cc mark_rsetless_slots, as device.cu publishes
// them. TEST INFRASTRUCTURE ONLY (built by tests/test_rsetless_emulation.py into its own .so; never part of
// libzgpu.so).
#include "emu_main.cc"

#include <set>

namespace {

struct HostClosure {
  uint16_t tgc = 0;
  uint32_t nsubj = 0;
  std::vector<uint32_t> row_ptr;
  std::vector<uint16_t> buf;  // the entries, padded, from the first 32-byte aligned element on
  const uint16_t* col = nullptr;
};

struct Indexed {
  Emu* e = nullptr;
  std::vector<HostClosure> cl;
  std::vector<uint8_t> blob;  // e->blob, with SF_NO_RSET marked when asked for
};

}  // namespace

extern "C" {

// Builds the index of every two-level pair of the published program; mark: set SF_NO_RSET as a publish does.
void* emu_index_create(void* h, int mark, int* n_marked) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return nullptr;
  Indexed* x = new Indexed();
  x->e = e;
  x->blob = e->blob;
  const DHeader* ph = reinterpret_cast<const DHeader*>(e->blob.data());
  const DStep* steps = reinterpret_cast<const DStep*>(e->blob.data() + ph->off_steps);
  std::vector<uint16_t> tgcs;
  for (uint32_t i = 0; i < ph->n_steps; ++i) {
    const DStep& st = steps[i];
    if (!(st.flags & kStepTargetL2) || std::find(tgcs.begin(), tgcs.end(), st.tgc) != tgcs.end()) continue;
    const uint16_t inner = e->sc.d_inv_cls[e->sc.d_type_inv[st.tstype].begin + st.tinv];
    const DCls &ci = e->h.cls[inner], &ct = e->h.cls[st.tgc];
    HostClosure c;
    c.tgc = st.tgc;
    c.nsubj = ci.nsubj;
    c.row_ptr.assign(c.nsubj + 1, 0);
    std::vector<uint16_t> ent;
    for (uint32_t u = 0; u < c.nsubj; ++u) {
      std::set<uint32_t> row;
      const uint64_t ri = ci.rrow_base + uint64_t(u) * ci.rstride;
      for (uint32_t a = e->h.rrow_ptr[ri]; a < e->h.rrow_ptr[ri + 1]; ++a) {
        const uint32_t g = e->h.rcol[a];
        if (g >= ct.nsubj) continue;
        const uint64_t rj = ct.rrow_base + uint64_t(g) * ct.rstride;
        for (uint32_t b = e->h.rrow_ptr[rj]; b < e->h.rrow_ptr[rj + 1]; ++b) row.insert(e->h.rcol[b]);
      }
      for (uint32_t t : row) ent.push_back(static_cast<uint16_t>(t));
      c.row_ptr[u + 1] = static_cast<uint32_t>(ent.size());
    }
    c.buf.assign(ent.size() + 16 + 16, 0);
    const size_t at = (32 - reinterpret_cast<uintptr_t>(c.buf.data()) % 32) % 32 / 2;
    std::copy(ent.begin(), ent.end(), c.buf.begin() + at);
    c.col = c.buf.data() + at;
    x->cl.push_back(std::move(c));
    tgcs.push_back(st.tgc);
  }
  *n_marked = mark && !tgcs.empty() ? mark_rsetless_slots(&x->blob, tgcs) : 0;
  return x;
}

void emu_index_destroy(void* x) { delete static_cast<Indexed*>(x); }

uint32_t emu_index_slot_flags(void* x, int slot) {
  const Indexed* d = static_cast<Indexed*>(x);
  const DHeader* ph = reinterpret_cast<const DHeader*>(d->blob.data());
  return reinterpret_cast<const DSlot*>(d->blob.data() + ph->off_slots)[slot].flags;
}

// One pass of check_kernel<COUNT, false, kMeet16> (pure permissions). raw = 0: the items' flags carry the hop depth.
// Returns the kernel's flags word; *bytes: the COUNT variant's algorithmic bytes.
uint32_t emu_index_check(void* x, const zg_check* items, uint64_t n, uint8_t* out, int raw, int count, uint64_t* bytes) {
  Indexed* d = static_cast<Indexed*>(x);
  Emu* e = d->e;
  KParams p{};
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.invert = 1;
  p.prog = d->blob.data();
  p.prog_bytes = static_cast<uint32_t>(d->blob.size());
  p.queries = items;
  p.nq = n;
  p.L = e->sc.max_leaves;
  p.out = out;
  p.final_codes = 1;
  Ctrl c;
  p.next = &c.next;
  p.subq_count = &c.subq_count;
  p.alg_bytes = &c.alg_bytes;
  p.flags = &c.flags;
  p.events = c.events;
  const uint32_t grid = 2, spill_cap = 4096;
  std::vector<uint4> spill(size_t(grid) * kWarpsPerBlock * spill_cap);
  std::vector<unsigned long long> memo(size_t(grid) * kWarpsPerBlock);
  std::vector<zg_check> subq(1 << 12);
  std::vector<uint32_t> subq_parent(1 << 12);
  p.spill = spill.data();
  p.spill_cap = spill_cap;
  p.subq = subq.data();
  p.subq_parent = subq_parent.data();
  p.subq_cap = subq.size();
  p.budget = 1 << 20;
  p.raw_items = raw;
  p.memo = memo.data();
  for (const auto& cl : d->cl) p.closure[p.n_closure++] = ClosureRef{cl.row_ptr.data(), cl.col, cl.nsubj, cl.tgc, 2};
  const size_t sm = p.prog_bytes + size_t(kWarpsPerBlock) * kWarpSmem;
  if (count) zg_emu::launch(check_kernel<true, false, kMeet16>, p, grid, kThreads, sm);
  else zg_emu::launch(check_kernel<false, false, kMeet16>, p, grid, kThreads, sm);
  *bytes = c.alg_bytes;
  return c.flags;
}

}  // extern "C"
