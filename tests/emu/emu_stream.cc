// emu_stream.cc -- streamed admission (kernels.cuh check_kernel<false, true, MEET>, wait_ready) with a real feed, under
// the CPU SIMT emulator (cuda_emu.h). device.cu check_host_multi copies a large call up in chunks on a copy stream and
// bumps the word the kernel polls behind each chunk, while one persistent grid already runs; here a "copy engine"
// thread lands the items chunk by chunk into a staging buffer that starts full of poison items (perm 0xFFFF: answer
// 255), publishing each new count with a release store. It lands a chunk only once the kernel has admitted a batch
// past what has landed (*p.next > landed), so that a warp waits at the frontier whenever a chunk lands: any item read
// before it landed answers 255. Only level 0 of a multi-pass program is streamed, and the halves of a split batch run
// unstreamed over the landed items, as device.cu check_device runs them. kMeet32 over the engine, or kMeetSet16 over
// emu_set.cc's host-built closure indexes, signatures and set tables. TEST INFRASTRUCTURE ONLY (built by
// tests/test_stream_emulation.py into its own .so; never part of libzgpu.so).
#include "emu_set.cc"

#include <chrono>
#include <cstring>
#include <thread>

namespace {

struct StreamRun {
  Emu* e = nullptr;
  Tabled* t = nullptr;  // nullptr: kMeet32 without closure indexes
  EmuOpts o{};
  uint64_t chunk = 1;
  uint64_t passes = 0, splits = 0, chunks = 0;
  uint32_t flags = 0;
};

const std::vector<uint8_t>& prog_of(const StreamRun& r) { return r.t ? r.t->s->x->blob : r.e->blob; }

// One launch of device.cu run_pass. feed != nullptr: q is the staging buffer and the pass is streamed from feed.
void stream_pass(StreamRun& r, const zg_check* q, uint64_t nq, uint8_t* val, uint8_t* out, bool raw, zg_check* subq,
                 uint32_t* subq_parent, uint64_t* n_sub, const zg_check* feed) {
  Emu* e = r.e;
  const std::vector<uint8_t>& blob = prog_of(r);
  KParams p{};
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = e->sc.has_expiry ? ptr(e->h.exp) : nullptr;
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.invert = r.o.invert;
  p.prog = blob.data();
  p.prog_bytes = static_cast<uint32_t>(blob.size());
  p.queries = q;
  p.nq = nq;
  p.L = e->sc.max_leaves;
  p.val = val;
  p.out = out;
  p.final_codes = 1;
  Ctrl c;
  c.ready = 0;
  p.next = &c.next;
  p.subq_count = &c.subq_count;
  p.alg_bytes = &c.alg_bytes;
  p.flags = &c.flags;
  p.events = c.events;
  p.ready = feed ? &c.ready : nullptr;
  const uint32_t grid = r.o.grid ? r.o.grid : 2;
  const size_t warps = size_t(grid) * kWarpsPerBlock;
  std::vector<uint4> spill(warps * r.o.spill_cap);
  std::vector<unsigned long long> memo(warps * std::max<uint32_t>(r.o.memo_entries, 1));
  p.spill = spill.data();
  p.spill_cap = r.o.spill_cap;
  p.subq = subq;
  p.subq_parent = subq_parent;
  p.subq_cap = subq ? r.o.subq_cap : 0;
  p.now = r.o.now;
  p.budget = r.o.budget;
  p.raw_items = raw;
  p.memo = memo.data();
  p.memo_entries = r.o.memo_entries;
  p.memo_after = r.o.memo_after;
  static const unsigned long long none = ~0ull;
  if (r.t) {
    const Signed* s = r.t->s;
    const Indexed* d = s->x;
    for (size_t i = 0; i < d->cl.size(); ++i) {
      const auto& cl = d->cl[i];
      const auto& sg = s->pairs[i];
      const auto& x = r.t->pairs[i];
      p.closure[p.n_closure++] = ClosureRef{cl.row_ptr.data(), cl.col, cl.nsubj, cl.tgc, 2, sg.sig.data(), sg.words,
                                            x.hdr.empty() ? &none : x.hdr.data(), x.tab.empty() ? &none : x.tab.data()};
    }
  }
  // the copy engine: chunk, count, chunk, count ... each chunk once a warp waits for it
  std::thread copier;
  bool kernel_done = false;  // a kernel that ends without admitting a batch past what has landed stops the feed
  if (feed) {
    zg_check* stage = const_cast<zg_check*>(q);
    copier = std::thread([&, stage] {
      uint64_t landed = 0;
      while (landed < nq) {
        while (__atomic_load_n(&c.next, __ATOMIC_ACQUIRE) <= landed && !__atomic_load_n(&kernel_done, __ATOMIC_ACQUIRE))
          std::this_thread::yield();
        if (__atomic_load_n(&kernel_done, __ATOMIC_ACQUIRE)) break;
        // the warp that took the batch is on its way into wait_ready: give it the time to get there
        std::this_thread::sleep_for(std::chrono::microseconds(100));
        const uint64_t end = std::min(nq, landed + r.chunk);
        std::memcpy(stage + landed, feed + landed, (end - landed) * sizeof(zg_check));
        __atomic_store_n(&c.ready, static_cast<unsigned long long>(end), __ATOMIC_RELEASE);
        landed = end;
        ++r.chunks;
      }
    });
  }
  const size_t sm = p.prog_bytes + size_t(kWarpsPerBlock) * kWarpSmem;
  if (feed) {
    if (r.t) zg_emu::launch(check_kernel<false, true, kMeetSet16>, p, grid, kThreads, sm);
    else zg_emu::launch(check_kernel<false, true>, p, grid, kThreads, sm);
    __atomic_store_n(&kernel_done, true, __ATOMIC_RELEASE);
    copier.join();
  } else {
    if (r.t) zg_emu::launch(check_kernel<false, false, kMeetSet16>, p, grid, kThreads, sm);
    else zg_emu::launch(check_kernel<false, false>, p, grid, kThreads, sm);
  }
  r.flags |= c.flags;
  if (n_sub) *n_sub = c.subq_count;
}

// device.cu check_device over host memory; feed: level 0 streamed into `items` (the staging buffer)
int stream_check(StreamRun& r, const zg_check* items, uint64_t n, uint8_t* out, const zg_check* feed) {
  if (n == 0) return 0;
  Emu* e = r.e;
  const uint32_t L = e->sc.max_leaves;
  if (!e->sc.has_nonpure) {
    stream_pass(r, items, n, nullptr, out, true, nullptr, nullptr, nullptr, feed);
    return 0;
  }
  std::vector<std::vector<zg_check>> q(1);
  std::vector<std::vector<uint32_t>> parent(1);
  std::vector<std::vector<uint8_t>> val;
  std::vector<uint64_t> nq;
  const zg_check* queries = items;
  uint64_t cur = n;
  bool raw = true;
  for (size_t lv = 0; cur > 0; ++lv) {
    if (lv > ZG_MAX_DEPTH + 1) return -2;
    nq.push_back(cur);
    val.emplace_back(cur * L + 4, 0);
    q.emplace_back(r.o.subq_cap);
    parent.emplace_back(r.o.subq_cap);
    uint64_t n_sub = 0;
    stream_pass(r, queries, cur, val[lv].data(), lv == 0 ? out : nullptr, raw, q[lv + 1].data(), parent[lv + 1].data(),
                &n_sub, lv == 0 ? feed : nullptr);
    if (n_sub > r.o.subq_cap) {
      // every item has landed: the streamed pass waited for all of them
      if (n < 2) return -3;
      ++r.splits;
      const uint64_t half = n / 2;
      int rc = stream_check(r, items, half, out, nullptr);
      if (rc) return rc;
      return stream_check(r, items + half, n - half, out + half, nullptr);
    }
    cur = n_sub;
    queries = q[lv + 1].data();
    raw = false;
    if (cur) ++r.passes;
  }
  if (nq.size() > 1) {
    struct FoldArgs {
      const uint8_t* prog;
      const zg_check* queries;
      unsigned long long n;
      uint32_t L;
      const uint8_t* val;
      uint8_t* out;
      const uint32_t* parent;
      uint8_t* parent_val;
    };
    for (size_t lv = nq.size(); lv-- > 0;) {
      FoldArgs a{prog_of(r).data(), lv == 0 ? items : q[lv].data(), nq[lv], L, val[lv].data(), lv == 0 ? out : nullptr,
                 lv == 0 ? nullptr : parent[lv].data(), lv == 0 ? nullptr : val[lv - 1].data()};
      zg_emu::launch(+[](const FoldArgs& f) { fold_kernel(f.prog, f.queries, f.n, f.L, f.val, f.out, f.parent, f.parent_val, 0); },
                     a, static_cast<unsigned>((nq[lv] + 255) / 256), 256, 0);
    }
  }
  return 0;
}

}  // namespace

extern "C" {

// Answers items[0, n) with level 0 streamed in chunks of `chunk` items: check_kernel<false, true> (kMeet32) over the
// engine h, or, with tabled (emu_set_create, every pair tabled), check_kernel<false, true, kMeetSet16> over its closure
// indexes. stats[0..2]: passes after level 0, split batches, chunks landed. Returns the kernels' flags word, or ~0u
// when the check failed (depth cap, a split of one item, a pair without a table).
uint32_t emu_stream_check(void* h, void* tabled, const zg_check* items, uint64_t n, uint8_t* out, const EmuOpts* o,
                          uint64_t chunk, uint64_t* stats) {
  StreamRun r;
  r.e = static_cast<Emu*>(h);
  r.t = static_cast<Tabled*>(tabled);
  r.o = *o;
  r.chunk = chunk ? chunk : 1;
  if (!r.e->published || (r.t && (r.t->s->x->e != r.e || emu_set_meet(r.t) != kMeetSet16))) return ~0u;
  zg_check poison{};
  poison.perm = 0xFFFF;
  poison.srel = 0xFFFF;
  std::vector<zg_check> stage(n, poison);
  const int rc = stream_check(r, stage.data(), n, out, items);
  stats[0] = r.passes;
  stats[1] = r.splits;
  stats[2] = r.chunks;
  return rc ? ~0u : r.flags;
}

}  // extern "C"
