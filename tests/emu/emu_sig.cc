// emu_sig.cc -- the check kernel's signature meet (kernels.cuh sig_meet, MEET = kMeetSig16 / kMeetSig32) under the CPU
// SIMT emulator (cuda_emu.h): emu_rset.cc's host-built closure indexes, plus the signature of every row as build.cu
// gpu_build_closure_sig writes it, and the entries widened to 32 bits for the kMeetSig32 instantiation. TEST
// INFRASTRUCTURE ONLY (built by tests/test_closure_sig_emulation.py into its own .so; never part of libzgpu.so).
#include "emu_rset.cc"

namespace {

struct Signed {
  Indexed* x = nullptr;
  int width = 2;
  struct Pair {
    uint32_t words = 0;
    std::vector<unsigned long long> sig;
    std::vector<uint32_t> wide;  // the entries at 32 bits (width 4)
  };
  std::vector<Pair> pairs;
};

}  // namespace

extern "C" {

// Signatures of every pair of the index x (emu_index_create): `words` 64-bit words per row, or with words = 0 the
// fewest with 64 * words >= 12 x the mean row length, at most 32 (as a publish chooses). width 4: the kernel reads
// 32-bit entries.
void* emu_sig_create(void* x, int width, uint32_t words) {
  Indexed* d = static_cast<Indexed*>(x);
  Signed* s = new Signed();
  s->x = d;
  s->width = width;
  for (const auto& c : d->cl) {
    Signed::Pair q;
    const uint64_t entries = c.row_ptr[c.nsubj];
    q.words = words;
    if (!q.words) {
      q.words = 1;
      while (q.words < 32 && 64ull * q.words * c.nsubj < 12ull * entries) q.words <<= 1;
    }
    const uint32_t lg = static_cast<uint32_t>(__builtin_ctz(q.words));
    q.sig.assign(size_t(c.nsubj) << lg, 0);
    for (uint32_t u = 0; u < c.nsubj; ++u)
      for (uint32_t a = c.row_ptr[u]; a < c.row_ptr[u + 1]; ++a)
        q.sig[(size_t(u) << lg) + sig_word(c.col[a], lg)] |= sig_mask(c.col[a]);
    q.wide.assign(c.col, c.col + entries);
    s->pairs.push_back(std::move(q));
  }
  return s;
}

void emu_sig_destroy(void* s) { delete static_cast<Signed*>(s); }

uint32_t emu_sig_words(void* s, int pair) { return static_cast<Signed*>(s)->pairs[pair].words; }

uint32_t emu_sig_rows(void* s, int pair) { return static_cast<Signed*>(s)->x->cl[pair].nsubj; }

// Row-major signature words of `pair` (rows x emu_sig_words).
void emu_sig_copy(void* s, int pair, unsigned long long* out) {
  const auto& q = static_cast<Signed*>(s)->pairs[pair];
  std::copy(q.sig.begin(), q.sig.end(), out);
}

// One pass of check_kernel<COUNT, false, kMeetSig16 / kMeetSig32> (pure permissions), as emu_index_check.
uint32_t emu_sig_check(void* sp, const zg_check* items, uint64_t n, uint8_t* out, int raw, int count, uint64_t* bytes) {
  Signed* s = static_cast<Signed*>(sp);
  Indexed* d = s->x;
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
  for (size_t i = 0; i < d->cl.size(); ++i) {
    const auto& cl = d->cl[i];
    const auto& q = s->pairs[i];
    const void* col = s->width == 2 ? static_cast<const void*>(cl.col) : static_cast<const void*>(q.wide.data());
    p.closure[p.n_closure++] = ClosureRef{cl.row_ptr.data(), col, cl.nsubj, cl.tgc, static_cast<uint16_t>(s->width),
                                          q.sig.empty() ? nullptr : q.sig.data(), q.words};
  }
  const size_t sm = p.prog_bytes + size_t(kWarpsPerBlock) * kWarpSmem;
  if (s->width == 2) {
    if (count) zg_emu::launch(check_kernel<true, false, kMeetSig16>, p, grid, kThreads, sm);
    else zg_emu::launch(check_kernel<false, false, kMeetSig16>, p, grid, kThreads, sm);
  } else {
    if (count) zg_emu::launch(check_kernel<true, false, kMeetSig32>, p, grid, kThreads, sm);
    else zg_emu::launch(check_kernel<false, false, kMeetSig32>, p, grid, kThreads, sm);
  }
  *bytes = c.alg_bytes;
  return c.flags;
}

}  // extern "C"
