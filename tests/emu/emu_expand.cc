// emu_expand.cc -- ExpandPermissionTree's kernels (expand.cuh) and Device::expand's launch sequence under the CPU SIMT
// emulator. TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_expand.py into its own .so; never part of libzgpu.so). The
// emulator driver emu_main.cc is compiled into this translation unit unchanged: its engine model (the product's schema
// compiler with its templates, the store and the host snapshot) comes with it. Added here: the level loop of
// Device::expand over host memory, a host exclusive sum in place of CUB's.
#include "emu_main.cc"

#include "../../spicedb-kubeapi-proxy_b200/csrc/expand.cuh"

// The trees of the n requests at clock `now`, as zg_expand_permission_trees returns them. threads: threads per block of
// both launches (any multiple of 32). info: [0] levels, [1] the largest warps per job of a level. Returns 0; -1 (not
// published, unknown slot or oversized template), -7 (a buffer is short: *n_nodes / *n_subjects = the sizes), -8 (cap).
extern "C" int emu_expand(void* h, const zg_expand_request* reqs, uint64_t n, uint32_t now, uint64_t cap, uint32_t threads,
                          int32_t* status, zg_expand_node* nodes_out, uint64_t node_cap, uint64_t* n_nodes_out,
                          zg_expand_subject* subj_out, uint64_t subj_cap, uint64_t* n_subj_out, uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  const Schema& sc = e->sc;
  info[0] = info[1] = 0;
  std::vector<XJob> jobs(n), next;
  unsigned long long mask = 0;
  for (uint64_t i = 0; i < n; ++i) {
    if (reqs[i].perm >= sc.slots.size() || !sc.x_ok[reqs[i].perm]) return -1;
    const uint32_t root = sc.x_root[reqs[i].perm];
    jobs[i] = XJob{static_cast<uint32_t>(i), UINT32_MAX, 0, reqs[i].res, root, 0};
    mask |= 1ull << sc.x_nodes[root].ncount;
  }
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  std::vector<uint32_t> failed(n, 0);
  std::vector<zg_expand_node> nodes;
  std::vector<zg_expand_subject> subj;
  XParams p{};
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = sc.has_expiry ? ptr(e->h.exp) : nullptr;
  p.rels = e->h.rels.data();
  p.cls = e->h.cls.data();
  p.nodes = sc.x_nodes.data();
  p.tgts = ptr(sc.x_tgts);
  p.counted = ptr(sc.x_counted);
  p.now = now;
  p.failed = failed.data();
  p.next_mask = &mask;
  uint64_t n_nodes = 0, n_subj = 0;
  while (!jobs.empty()) {
    p.m = expand_warps(mask);
    info[1] = std::max<uint64_t>(info[1], p.m);
    if (n_nodes + n_subj + jobs.size() * p.m > cap) return -8;
    const uint64_t N = jobs.size() * p.m;
    std::vector<unsigned long long> cnt(3 * N + 1, 0), off(3 * N + 1, 0);
    p.jobs = jobs.data();
    p.n_jobs = jobs.size();
    p.cnt = cnt.data();
    p.off = off.data();
    const unsigned blocks = static_cast<unsigned>((N * 32 + threads - 1) / threads);
    zg_emu::launch(expand_count_kernel, p, blocks, threads, 0);
    for (uint64_t i = 1; i <= 3 * N; ++i) off[i] = off[i - 1] + cnt[i - 1];
    const uint64_t lvl_nodes = off[N], lvl_subj = off[2 * N] - off[N], n_next = off[3 * N] - off[2 * N];
    if (n_nodes + lvl_nodes + n_subj + lvl_subj + n_next > cap) return -8;
    nodes.resize(n_nodes + lvl_nodes);
    subj.resize(n_subj + lvl_subj);
    next.assign(n_next, XJob{});
    p.node_base = n_nodes;
    p.subj_base = n_subj;
    p.out_nodes = nodes.data();
    p.out_subj = subj.data();
    p.next = next.data();
    mask = 0;
    zg_emu::launch(expand_emit_kernel, p, blocks, threads, 0);
    n_nodes += lvl_nodes;
    n_subj += lvl_subj;
    jobs.swap(next);
    ++info[0];
  }
  for (uint64_t i = 0; i < n; ++i) status[i] = failed[i] ? ZG_EDEPTH : ZG_OK;
  expand_drop_failed(failed, &nodes, &subj);
  *n_nodes_out = nodes.size();
  *n_subj_out = subj.size();
  if (nodes.size() > node_cap || subj.size() > subj_cap) return -7;
  std::copy(nodes.begin(), nodes.end(), nodes_out);
  std::copy(subj.begin(), subj.end(), subj_out);
  return 0;
}
