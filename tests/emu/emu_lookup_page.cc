// emu_lookup_page.cc -- the kernels of a LookupResources page (kernels.cuh lookup_select_kernel, lookup_bound_kernel,
// lookup_window_kernel) under the CPU SIMT emulator, driven by a restatement of device.cu Device::lookup_page's loop
// over host memory: select (or bound) and sort, then windows verified by the emulated check and scanned in id order.
// TEST INFRASTRUCTURE ONLY (built by tests/test_lookup_page_emulation.py into its own .so; never part of libzgpu.so).
// The candidate list comes from the caller: the walk and the flat union are the product's, tested elsewhere.
#include "emu_main.cc"

extern "C" {

// cand[0, n): the candidates (sorted: ascending without repeats, as the exhaustive list; flat: every one is an answer,
// repeats allowed, no verification). info: [0] answers found, [1] candidates after the cursor, [2] verified, [3]
// windows, [4] launches. Returns 0, -3 (ZG_EDEPTH), or another negative code of the emulated check.
int emu_lookup_page(void* h, uint16_t res_type, const zg_check* proto_in, int has_after, uint32_t after, uint64_t want,
                    uint32_t self, uint64_t first_w, uint32_t growth, const uint32_t* cand, uint64_t n, int sorted, int flat,
                    const EmuOpts* o, uint32_t* out, uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  (void)res_type;
  const zg_check proto = *proto_in;
  for (int k = 0; k < 5; ++k) info[k] = 0;
  unsigned long long ctrl[3] = {0, 0, 0};
  std::vector<uint32_t> sel_buf(n + 2), sorted_buf;
  const uint32_t* sel = cand;
  uint64_t m = n;
  uint32_t quiet = ZG_NO_OBJECT;
  if (sorted) {
    if (has_after && n) {
      struct BArgs {
        const uint32_t* ids;
        unsigned long long n;
        uint32_t after;
        unsigned long long* at;
      } ba{cand, n, after, ctrl + 2};
      zg_emu::launch(+[](const BArgs& a) { lookup_bound_kernel(a.ids, a.n, a.after, a.at); }, ba, 1, 1, 0);
      ++info[4];
      sel = cand + ctrl[2];
      m = n - ctrl[2];
    }
  } else {
    const uint64_t n_sel = n + (self != ZG_NO_OBJECT ? 1 : 0);
    struct SArgs {
      const uint32_t* cand;
      unsigned long long n;
      uint32_t has_after, after, self;
      uint32_t* out;
      unsigned long long* ctrl;
    } sa{cand, n, has_after ? 1u : 0u, after, self, sel_buf.data(), ctrl};
    if (n_sel) {
      zg_emu::launch(+[](const SArgs& a) { lookup_select_kernel(a.cand, a.n, a.has_after, a.after, a.self, a.out, a.ctrl); },
                     sa, static_cast<unsigned>((n_sel + 255) / 256), 256, 0);
      ++info[4];
    }
    m = ctrl[0];
    if (self != ZG_NO_OBJECT && !ctrl[1]) quiet = self;
    sorted_buf.assign(sel_buf.begin(), sel_buf.begin() + static_cast<long>(m));
    std::sort(sorted_buf.begin(), sorted_buf.end());  // sort_u32
    sorted_buf.push_back(0);
    sel = sorted_buf.data();
  }
  info[1] = m;
  if (m == 0) return 0;
  ctrl[0] = ctrl[1] = 0;
  struct WArgs {
    const uint32_t* ids;
    unsigned long long n;
    uint32_t has_prev;
    const uint8_t* codes;
    uint32_t quiet;
    unsigned long long want;
    uint32_t* out;
    unsigned long long* ctrl;
  };
  auto window = [&](const WArgs& a) {
    zg_emu::launch(+[](const WArgs& w) { lookup_window_kernel(w.ids, w.n, w.has_prev, w.codes, w.quiet, w.want, w.out, w.ctrl); },
                   a, 1, kWindowThreads, 0);
    ++info[4];
  };
  if (flat) {
    window(WArgs{sel, m, 0, nullptr, ZG_NO_OBJECT, want, out, ctrl});
    info[0] = ctrl[0];
    return 0;
  }
  uint64_t pos = 0, w = std::max<uint64_t>(first_w, 2 * want);
  for (;;) {
    w = std::min(w, m - pos);
    std::vector<zg_check> jobs(w);
    std::vector<uint8_t> codes(w);
    for (uint64_t i = 0; i < w; ++i) {  // lookup_fill_kernel
      jobs[i] = proto;
      jobs[i].res = sel[pos + i];
    }
    e->flags = 0;
    if (int rc = check(e, *o, jobs.data(), w, codes.data(), false)) return rc;
    window(WArgs{sel + pos, w, pos > 0 ? 1u : 0u, codes.data(), quiet, want, out, ctrl});
    ++info[3];
    info[2] += w;
    if (ctrl[1]) return -3;
    pos += w;
    info[0] = ctrl[0];
    if (ctrl[0] >= want || pos == m) break;
    const uint64_t left = m - pos;
    uint64_t next = std::min<uint64_t>(left, w * growth);
    if (ctrl[0]) {
      const double est = static_cast<double>(want - ctrl[0]) * static_cast<double>(pos) / static_cast<double>(ctrl[0]) * 1.25;
      next = est >= static_cast<double>(left) ? left : std::max<uint64_t>(next, static_cast<uint64_t>(est) + 1);
    }
    w = next;
  }
  return 0;
}

}  // extern "C"
