// device.cu -- snapshot upload and the launch sequences of the hot path.
//
// Call graph it replaces in the reference:
//   CheckBulkPermissions (pkg/authz/check.go:48, postfilter.go:134) -> check_*()
//   LookupResources      (pkg/authz/lookups.go:65)                    -> lookup()
//   LookupSubjects       (v1 API, no proxy call site)                 -> lookup_subjects()
#include "device.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>

#include <cub/cub.cuh>

#include "expand.cuh"
#include "filter.cuh"
#include "import.cuh"
#include "ingress.cuh"
#include "kernels.cuh"

namespace zg {

#define ZG_CUDA(expr)                                                                   \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      if (err) *err = std::string(#expr) + ": " + cudaGetErrorString(_e);               \
      return ZG_ECUDA;                                                                  \
    }                                                                                   \
  } while (0)

#define ZG_STR2(x) #x
#define ZG_STR(x) ZG_STR2(x)
const char* build_info() {
  return "libzgpu sm_90a built " __DATE__ " " __TIME__ " STACK_CAP=" ZG_STR(ZG_STACK_CAP) " RSET_CAP=" ZG_STR(ZG_RSET_CAP) " MIN_BLOCKS=" ZG_STR(ZG_MIN_BLOCKS);
}

// zg_import_relationships' scratch (import.cuh): the staged call, the new-name table, the items' tuples and keys.
struct Device::ImportScratch {
  DevBuf groups, blob, offs, tables;
  DevBuf slots, first, hash, slot_type, occ_id, occ_slot;
  DevBuf new_keys, new_vals, new_keys2, new_vals2, slot_tmp, out_hash, extent, type_start;
  DevBuf tuples, key_hi, key_lo, key_hi2, key_lo2, vals, vals2, known;
  DevBuf ctrl;  // [0] bad, [1] dup, [2] found, [3] new names
  DevBuf cub, ids, base, rtype_of_rel;
  uint64_t n = 0;
  uint32_t n_groups = 0;
  ~ImportScratch() {
    for (DevBuf* b : {&groups, &blob, &offs, &tables, &slots, &first, &hash, &slot_type, &occ_id, &occ_slot, &new_keys,
                      &new_vals, &new_keys2, &new_vals2, &slot_tmp, &out_hash, &extent, &type_start, &tuples, &key_hi,
                      &key_lo, &key_hi2, &key_lo2, &vals, &vals2, &known, &ctrl, &cub, &ids, &base, &rtype_of_rel})
      b->release();
  }
};

void Device::ImportScratchFree::operator()(ImportScratch* x) const { delete x; }

bool DevBuf::ensure(size_t bytes) {
  if (bytes <= cap) return true;
  release();
  size_t want = std::max<size_t>(bytes, 256);
  if (cudaMalloc(&p, want) != cudaSuccess) {
    p = nullptr;
    cap = 0;
    cudaGetLastError();
    return false;
  }
  cap = want;
  return true;
}
void DevBuf::release() {
  if (p) cudaFree(p);
  p = nullptr;
  cap = 0;
}
Snapshot::~Snapshot() {
  row_ptr.release();
  col.release();
  exp.release();
  prog.release();
  rrow_ptr.release();
  rcol.release();
  col_alt.release();
  exp_alt.release();
  rcol_alt.release();
  type_bit_base.release();
  for (auto& r : resources) r.release();
  for (auto& f : flat_cls) f.release();
  ls_fwd.release();
  ls_type_off.release();
  ls_mask.release();
  for (DevBuf* b : {&x_nodes, &x_tgts, &x_counted, &x_rels, &x_cls}) b->release();
  for (auto& c : closure) {
    c.row_ptr.release();
    c.col.release();
    c.sig.release();
    c.set_hdr.release();
    c.set_tab.release();
  }
  for (auto& r : records) r.rec.release();
}

Device::~Device() {
  if (stream) cudaStreamSynchronize(stream);
  snap.reset();
  spill_.release();
  ctrl_.release();
  memo_.release();
  flat_ctrl_.release();
  flat_idx_.release();
  for (auto* v : {&q_, &parent_, &val_})
    for (auto& b : *v) b.release();
  stage_in_.release();
  stage_out_.release();
  route_ctrl_.release();
  lk_jobs_.release();
  lk_codes_.release();
  lk_ids_.release();
  rb_visited_.release();
  rb_front_[0].release();
  rb_front_[1].release();
  rb_cand_.release();
  for (auto* b : {&lb_params_, &lb_owner_, &lb_ctrl_, &lb_keys_[0], &lb_keys_[1]}) b->release();
  for (auto* b : {&ls_jobs_, &ls_codes_, &ls_has_, &ls_ids_, &ls_ctrl_}) b->release();
  for (auto* b : {&flt_out_, &flt_exp_, &flt_ctrl_, &mention_bits_}) b->release();
  for (auto& l : pl_)
    for (auto* b : {&l.in, &l.val, &l.out, &l.raised, &l.parent, &l.pos}) b->release();
  for (auto* b : {&home_, &home_pos_, &home_out_, &peer_ctrl_}) b->release();
  for (auto* b : {&hl.front[0], &hl.front[1], &hl.next, &hl.items, &hl.codes, &hl.routed, &hl.keys, &hl.ids}) b->release();
  if (pin_peer_) cudaFreeHost(pin_peer_);
  for (cudaEvent_t ev : ev_peer_)
    if (ev) cudaEventDestroy(ev);
  if (pin_in_) cudaFreeHost(pin_in_);
  if (pin_out_) cudaFreeHost(pin_out_);
  if (pin_ready_) cudaFreeHost(pin_ready_);
  if (pin_lk_) cudaFreeHost(pin_lk_);
  if (cstream_) {
    cudaStreamSynchronize(cstream_);
    cudaStreamDestroy(cstream_);
  }
  if (ev_reset_) cudaEventDestroy(ev_reset_);
  if (ev0_) cudaEventDestroy(ev0_);
  if (ev1_) cudaEventDestroy(ev1_);
  if (last_done_) cudaEventDestroy(last_done_);
  if (stream) cudaStreamDestroy(stream);
}

static size_t smem_bytes(uint32_t prog_bytes) {
  return prog_bytes + static_cast<size_t>(kWarpsPerBlock) * kWarpSmem;
}

std::string Device::init(int dev, uint64_t subq_cap, uint32_t budget) {
  if (const char* v = std::getenv("ZGPU_NO_INVERT")) invert = !(*v && *v != '0');
  if (const char* v = std::getenv("ZGPU_NO_RBFS")) use_rbfs = !(*v && *v != '0');
  if (const char* v = std::getenv("ZGPU_LOOKUP_BATCH_CAP")) lb_cap_ = std::max<uint64_t>(1024, std::strtoull(v, nullptr, 10));
  if (const char* v = std::getenv("ZGPU_LOOKUP_PAGE_WINDOW")) lp_first_ = std::max<uint64_t>(1, std::strtoull(v, nullptr, 10));
  if (const char* v = std::getenv("ZGPU_LOOKUP_PAGE_GROWTH"))
    lp_growth_ = std::max<uint32_t>(2, static_cast<uint32_t>(std::strtoul(v, nullptr, 10)));
  if (const char* v = std::getenv("ZGPU_CLOSURE_CAP")) closure_cap_ = std::strtoull(v, nullptr, 10);  // tests: 0 = no index
  if (const char* v = std::getenv("ZGPU_CLOSURE_SIG_WORDS"))  // tests: 0 = no signatures, 1 = one word (most tests maybe)
    closure_sig_words_ = static_cast<uint32_t>(std::strtoul(v, nullptr, 10));
  if (const char* v = std::getenv("ZGPU_CLOSURE_TABLE")) closure_table_ = !(*v == '0' && !v[1]);  // tests: 0 = no tables
  if (const char* v = std::getenv("ZGPU_FLAT_CHECK")) flat_check_ = !(*v == '0' && !v[1]);  // tests, A/B: 0 = no SF_FLAT
  if (const char* v = std::getenv("ZGPU_FLAT_RECORDS")) flat_records_ = !(*v == '0' && !v[1]);  // tests, A/B: 0 = none
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") +
           " (libzgpu has no CPU fallback)";
  if (dev < 0) {
    if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  }
  if (dev >= count) return "CUDA device ordinal out of range";
  if ((e = cudaSetDevice(dev)) != cudaSuccess) return std::string("cudaSetDevice: ") + cudaGetErrorString(e);
  device = dev;
  cudaDeviceProp prop{};
  if ((e = cudaGetDeviceProperties(&prop, dev)) != cudaSuccess)
    return std::string("cudaGetDeviceProperties: ") + cudaGetErrorString(e);
  sm_count_ = prop.multiProcessorCount;
  if ((e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)) != cudaSuccess)
    return std::string("cudaStreamCreate: ") + cudaGetErrorString(e);
  cudaEventCreate(&ev0_);
  cudaEventCreate(&ev1_);
  cudaEventCreateWithFlags(&last_done_, cudaEventDisableTiming);
  if ((e = cudaStreamCreateWithFlags(&cstream_, cudaStreamNonBlocking)) != cudaSuccess)
    return std::string("cudaStreamCreate: ") + cudaGetErrorString(e);
  cudaEventCreateWithFlags(&ev_reset_, cudaEventDisableTiming);
  if (subq_cap) subq_cap_ = subq_cap;
  if (budget) budget_ = budget;
  if (!ctrl_.ensure(128) || !flat_ctrl_.ensure(16)) return "out of device memory";
  cudaMemset(ctrl_.p, 0, 128);
  cudaMemset(flat_ctrl_.p, 0, 16);
  return "";
}

std::string Device::publish(const HostSnapshot& h, const Schema& sc, uint64_t revision) {
  cudaSetDevice(device);
  closure_ms = 0;
  auto s = std::make_shared<Snapshot>();
  auto up = [&](DevBuf& b, const void* src, size_t bytes) -> bool {
    if (!b.ensure(bytes + 64)) return false;  // + 64: rows are streamed with aligned 128-bit loads (build.cu)
    if (bytes && cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, stream) != cudaSuccess) return false;
    s->bytes += bytes;
    return true;
  };
  bool ok = up(s->row_ptr, h.row_ptr.data(), h.row_ptr.size() * 4) && up(s->col, h.col.data(), h.col.size() * 4) &&
            up(s->rrow_ptr, h.rrow_ptr.data(), h.rrow_ptr.size() * 4) && up(s->rcol, h.rcol.data(), h.rcol.size() * 4);
  if (ok && sc.has_expiry) ok = up(s->exp, h.exp.data(), h.exp.size() * 4);
  s->resources.resize(h.resources.size());
  s->n_resources.resize(h.resources.size());
  for (size_t t = 0; ok && t < h.resources.size(); ++t) {
    s->n_resources[t] = h.resources[t].size();
    ok = up(s->resources[t], h.resources[t].data(), h.resources[t].size() * 4);
  }
  if (!ok || cudaStreamSynchronize(stream) != cudaSuccess)
    return std::string("snapshot upload failed: ") + cudaGetErrorString(cudaGetLastError());
  s->n_tuples = h.n_tuples;
  return finish_publish(s, h, sc, revision);
}

std::string Device::publish_gpu(const Store& store, const Schema& sc, uint64_t revision, bool verify) {
  cudaSetDevice(device);
  closure_ms = 0;
  HostSnapshot lay = store.layout();
  auto s = std::make_shared<Snapshot>();
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0, stream);
  std::string err = gpu_build_snapshot(store, sc, &lay, stream, s.get(), own_rank, own_count);
  cudaEventRecord(e1, stream);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  last_build_ms = ms;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (!err.empty()) return "GPU snapshot build failed: " + err;
  ++full_publishes;
  if (verify) {
    std::string verr = verify_snapshot(*s, store, sc, &lay);
    if (!verr.empty()) return verr;
  }
  return finish_publish(s, lay, sc, revision);
}

// test mode (ZGPU_VERIFY_BUILD=1): the host builder must produce byte-identical arrays
std::string Device::verify_snapshot(Snapshot& sn, const Store& store, const Schema& sc, const HostSnapshot* lay) {
  Snapshot* s = &sn;
  if (s->resources_stale) {
    std::string rerr = gpu_resource_lists(s, stream);
    if (!rerr.empty()) return rerr;
  }
  cudaStreamSynchronize(stream);
  HostSnapshot h = store.build(own_rank, own_count);
  if (!h.err.empty()) return h.err;
  auto same = [&](const DevBuf& d, const std::vector<uint32_t>& v, const char* what) -> std::string {
    std::vector<uint32_t> got(v.size());
    if (!v.empty() && cudaMemcpy(got.data(), d.p, v.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
      return std::string("verify: cannot read ") + what;
    for (size_t i = 0; i < v.size(); ++i)
      if (got[i] != v[i])
        return std::string("verify: ") + what + " differs at " + std::to_string(i) + " (gpu " + std::to_string(got[i]) +
               ", host " + std::to_string(v[i]) + ")";
    return "";
  };
  if (h.n_tuples != s->n_tuples) return "verify: relationship count differs";
  for (auto m : {same(s->row_ptr, h.row_ptr, "row_ptr"), same(s->col, h.col, "col"), same(s->rrow_ptr, h.rrow_ptr, "rrow_ptr"),
                 same(s->rcol, h.rcol, "rcol"), sc.has_expiry ? same(s->exp, h.exp, "exp") : std::string()})
    if (!m.empty()) return m;
  for (size_t t = 0; t < h.resources.size(); ++t) {
    if (h.resources[t].size() != s->n_resources[t]) return "verify: resource list size differs";
    std::string m = same(s->resources[t], h.resources[t], "resources");
    if (!m.empty()) return m;
  }
  for (size_t c = 0; c < h.cls.size(); ++c) {
    const bool empty = lay ? (lay->cls[c].flags & CF_EMPTY) != 0 : s->cls_count[c] == 0;
    if (((h.cls[c].flags & CF_EMPTY) != 0) != empty) return "verify: class emptiness differs";
  }
  return "";
}
std::string Device::verify_against_host(const Store& store, const Schema& sc) {
  std::shared_ptr<Snapshot> s = snap;
  if (!s) return "verify: no snapshot";
  cudaSetDevice(device);
  return verify_snapshot(*s, store, sc, nullptr);
}

std::string Device::publish_delta(const Store& store, const Schema& sc, uint64_t revision) {
  std::shared_ptr<Snapshot> s = snap;
  // an engine that is one shard of a store per process (shard_count > 1 over a store of its own) always rebuilds
  const bool own_store_shard = shard_count > 1 && own_count < 2;
  if (!s || !s->delta_ok || !store.journal_ok || own_store_shard || store.journal.size() > Store::kMaxJournal || !store.layout_stable())
    return "full";
  cudaSetDevice(device);
  closure_ms = 0;
  HostSnapshot lay = store.layout();  // same capacities as the resident snapshot: same bases
  if (lay.n_objects != s->n_objects) return "full";
  // readers on other streams (zg_check_bulk_device) are ordered through last_done_
  if (have_last_ && cudaStreamWaitEvent(stream, last_done_, 0) != cudaSuccess) return "full";
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0, stream);
  std::vector<uint32_t> cls_delta;
  std::string err = gpu_apply_delta(store, sc, lay, stream, s.get(), &cls_delta, own_rank, own_count);
  const uint64_t failures = closure_failures;
  if (err.empty() && (!s->closure.empty() || !s->records.empty())) {
    // a closure index or range records whose classes this write changed are rebuilt from the merged rows before
    // anybody reads the snapshot again: stale ones are never read
    std::vector<uint8_t> touched(lay.cls.size(), 0);
    for (const auto& j : store.journal) {
      const int k = sc.class_of(j.t.rel, j.t.stype, j.t.srel);
      if (k >= 0) touched[lay.rels[sc.slots[j.t.rel].rel_index].cls_begin + k] = 1;
    }
    if (!s->closure.empty()) build_closures(s.get(), lay, &touched);
    build_flat_records(s.get(), &touched);
  }
  cudaEventRecord(e1, stream);
  cudaEventRecord(last_done_, stream);
  have_last_ = true;
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  last_build_ms = ms;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (!err.empty()) {
    snap.reset();  // the arrays may be half merged: nobody may read them; the caller rebuilds
    return err == "relayout" || err == "corrupt" ? "full" : err;
  }
  // a pair that lost its index (a failed rebuild) republishes the program: its slots' SF_NO_RSET flags are recomputed
  bool structural = closure_failures != failures;
  for (size_t c = 0; c < cls_delta.size(); ++c) {
    const uint64_t before = s->cls_count[c];
    s->cls_count[c] = before + static_cast<int32_t>(cls_delta[c]);
    if ((before == 0) != (s->cls_count[c] == 0)) structural = true;
  }
  s->resources_stale = true;
  s->revision = revision;
  ++delta_publishes;
  if (!structural) return "";
  // a class became empty or non-empty: the flattened steps of the program change
  for (size_t c = 0; c < lay.cls.size(); ++c)
    if (s->cls_count[c]) lay.cls[c].flags &= static_cast<uint16_t>(~CF_EMPTY);
  lay.n_tuples = s->n_tuples;
  return finish_publish(s, lay, sc, revision);
}

void Device::build_closures(Snapshot* s, const HostSnapshot& h, const std::vector<uint8_t>* rebuild) {
  const std::vector<DCls>& cls = h.cls;
  // One width for the whole snapshot, so that a kernel instantiation inlines one meet. Object ids of a type stay below
  // its capacity, and a write that grows a capacity lays the snapshot out again (a full publish).
  uint8_t width = 2;
  for (const auto& c : s->closure)
    if (h.n_objects[cls[c.tgc].rtype] > 65536u) width = 4;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  for (auto& c : s->closure) {
    if (c.width == width && (rebuild ? !((*rebuild)[c.inner] || (*rebuild)[c.tgc]) : c.done)) continue;
    c.width = width;
    if (!e0) {
      cudaEventCreate(&e0);
      cudaEventCreate(&e1);
    }
    cudaEventRecord(e0, stream);
    std::string err = gpu_build_closure(*s, cls[c.inner], cls[c.tgc], closure_cap_, &c, stream);
    cudaEventRecord(e1, stream);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    closure_ms += ms;
    c.done = true;
    if (!err.empty()) {
      // The index is optional: a build that fails (an allocation the budget did not foresee) leaves the pair without
      // one, and its steps meet through batch_l2. Nothing half built is ever handed to the kernel.
      c.built = false;
      c.entries = 0;
      c.row_ptr.release();
      c.col.release();
      c.sig.release();
      c.sig_words = 0;
      c.set_hdr.release();
      c.set_tab.release();
      c.set_built = false;
      cudaGetLastError();
      ++closure_failures;
      continue;
    }
    ++closure_builds;
    // The signatures are optional too: without them (over budget, or a failed build) the pair meets through
    // closure_meet over its index.
    cudaEventRecord(e0, stream);
    err = gpu_build_closure_sig(&c, closure_sig_words_, stream);
    cudaEventRecord(e1, stream);
    cudaEventSynchronize(e1);
    ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    closure_ms += ms;
    c.sig_ms = ms;
    if (!err.empty()) {
      c.sig.release();
      c.sig_words = 0;
      cudaGetLastError();
    }
    // And the set tables, for 16-bit indexes whose target type leaves 0xFFFF free to mark an empty slot: without them
    // sig_meet searches the row for each "maybe" (or, without signatures, the pair meets through closure_meet).
    const bool table = closure_table_ && width == 2 && h.n_objects[cls[c.tgc].rtype] < 65536u;
    cudaEventRecord(e0, stream);
    err = gpu_build_closure_table(&c, table ? kTableSeeds : 0u, stream);
    cudaEventRecord(e1, stream);
    cudaEventSynchronize(e1);
    ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    closure_ms += ms;
    c.set_ms = ms;
    if (!err.empty()) {
      c.set_hdr.release();
      c.set_tab.release();
      c.set_built = false;
      cudaGetLastError();
    }
  }
  if (e0) {
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
}

void Device::build_flat_records(Snapshot* s, const std::vector<uint8_t>* rebuild) {
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  for (auto& r : s->records) {
    if (rebuild && !(*rebuild)[r.gc]) continue;
    if (!e0) {
      cudaEventCreate(&e0);
      cudaEventCreate(&e1);
    }
    cudaEventRecord(e0, stream);
    std::string err = gpu_build_flat_records(*s, &r, stream);
    cudaEventRecord(e1, stream);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    r.ms = ms;
    if (!err.empty()) {  // the records are optional: the class's steps read the CSR
      r.built = false;
      r.rec.release();
      cudaGetLastError();
    }
  }
  if (e0) {
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
}

std::string Device::finish_publish(std::shared_ptr<Snapshot> s, const HostSnapshot& h, const Schema& sc, uint64_t revision) {
  std::vector<uint8_t> blob = sc.blob(h.rels, h.cls);
  auto up = [&](DevBuf& b, const void* src, size_t bytes) -> bool {
    if (!b.ensure(bytes ? bytes : 16)) return false;
    if (bytes && cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, stream) != cudaSuccess) return false;
    s->bytes += bytes;
    return true;
  };
  bool ok = up(s->prog, blob.data(), blob.size());
  {
    std::vector<unsigned long long> base(h.n_objects.size() + 1, 0);
    for (size_t t = 0; t < h.n_objects.size(); ++t) base[t + 1] = base[t] + ((uint64_t(h.n_objects[t]) + 31) & ~31ull);
    s->total_bits = base.back();
    s->n_objects = h.n_objects;
    s->rels = h.rels;
    s->cls = h.cls;
    if (ok) ok = up(s->type_bit_base, base.data(), base.size() * 8);
  }
  {
    std::vector<FwdClass> fwd;
    std::vector<uint32_t> type_off;
    sc.forward_tables(h.rels, &fwd, &type_off);
    s->ls_mask_words = sc.fwd_mask_words;
    if (ok) ok = up(s->ls_fwd, fwd.data(), fwd.size() * sizeof(FwdClass)) && up(s->ls_type_off, type_off.data(), type_off.size() * 4) &&
                 up(s->ls_mask, sc.fwd_mask.data(), sc.fwd_mask.size() * 4);
    if (ok) ok = up(s->x_nodes, sc.x_nodes.data(), sc.x_nodes.size() * sizeof(XNode)) &&
                 up(s->x_tgts, sc.x_tgts.data(), sc.x_tgts.size() * 4) && up(s->x_counted, sc.x_counted.data(), sc.x_counted.size() * 4) &&
                 up(s->x_rels, h.rels.data(), h.rels.size() * sizeof(DRel)) && up(s->x_cls, h.cls.data(), h.cls.size() * sizeof(DCls));
  }
  if (!ok || cudaStreamSynchronize(stream) != cudaSuccess)
    return std::string("snapshot upload failed: ") + cudaGetErrorString(cudaGetLastError());
  // flat-union slots: LookupResources is the union of the subject's reverse rows
  {
    const size_t ns = sc.slots.size();
    s->flat_cls.resize(ns);
    s->flat_n.assign(ns, -1);
    for (size_t sl = 0; ok && sl < ns; ++sl) {
      if (sc.d_slots[sl].kind == SK_NONPURE) continue;
      const DUnit& u = sc.d_units[sc.d_slots[sl].unit];
      bool flat = true;
      std::vector<FlatLookupClass> fc;
      for (int oi = u.op_begin; oi < u.op_end && flat; ++oi) {
        const DOp& op = sc.d_ops[oi];
        if (op.kind != OP_REL) { flat = false; break; }
        const DRel& r = h.rels[op.rel];
        for (uint16_t k = 0; k < r.ncls; ++k) {
          const DCls& c = h.cls[r.cls_begin + k];
          if (c.flags & CF_EMPTY) continue;
          if ((c.sslot != kNone && c.sslot != kWildcard) || (c.flags & CF_EXPIRY)) { flat = false; break; }
          fc.push_back(FlatLookupClass{c.rrow_base, c.nsubj, c.stype, static_cast<uint16_t>(c.sslot == kWildcard), c.rstride, 0});
        }
      }
      if (!flat) continue;
      s->flat_n[sl] = static_cast<int>(fc.size());
      ok = up(s->flat_cls[sl], fc.data(), fc.size() * sizeof(FlatLookupClass));
    }
    if (ok && cudaStreamSynchronize(stream) != cudaSuccess) ok = false;
    if (!ok) return std::string("snapshot upload failed (flat lookup tables)");
  }
  s->prog_bytes = static_cast<uint32_t>(blob.size());
  s->max_leaves = sc.max_leaves;
  s->has_nonpure = sc.has_nonpure;
  {
    const DHeader* ph = reinterpret_cast<const DHeader*>(blob.data());
    const DStep* steps = reinterpret_cast<const DStep*>(blob.data() + ph->off_steps);
    // the pairs of the two-level steps: a pair indexed by an earlier publish of this snapshot keeps its index (a write
    // that changed one of its classes has rebuilt it already, publish_delta). Only an unsharded engine with the
    // direction-optimised probes has any: a shard does not hold the subjects' reverse rows, and without the probes
    // nothing meets. An engine without pairs builds nothing, at publish or after a write.
    const bool indexable = invert && shard_count <= 1 && own_count <= 1;
    std::vector<Snapshot::Closure> pairs;
    for (uint32_t i = 0; i < ph->n_steps; ++i) {
      if (!(steps[i].flags & kStepTargetL2)) continue;
      s->has_l2 = true;
      if (!indexable) continue;
      const uint16_t inner = sc.d_inv_cls[sc.d_type_inv[steps[i].tstype].begin + steps[i].tinv], tgc = steps[i].tgc;
      bool seen = false;
      for (const auto& c : pairs) seen = seen || c.tgc == tgc;
      if (seen || pairs.size() == static_cast<size_t>(kMaxClosure)) continue;
      auto old = std::find_if(s->closure.begin(), s->closure.end(),
                              [&](const Snapshot::Closure& c) { return c.tgc == tgc && c.inner == inner; });
      if (old != s->closure.end()) {
        pairs.push_back(*old);
        old->row_ptr = DevBuf{};  // moved
        old->col = DevBuf{};
        old->sig = DevBuf{};
        old->set_hdr = DevBuf{};
        old->set_tab = DevBuf{};
      } else {
        pairs.emplace_back();
        pairs.back().inner = inner;
        pairs.back().tgc = tgc;
      }
    }
    for (auto& c : s->closure) {
      c.row_ptr.release();
      c.col.release();
      c.sig.release();
      c.set_hdr.release();
      c.set_tab.release();
    }
    s->closure = std::move(pairs);
    build_closures(s.get(), h, nullptr);
    // slots whose checks only meet over the indexes just built load no memberships at admission (kernels.cuh), and
    // those of them whose meets all have signatures and set tables are answered by flat_check_kernel
    std::vector<uint16_t> indexed, tabled;
    for (const auto& c : s->closure)
      if (c.built) {
        indexed.push_back(c.tgc);
        if (c.sig_words && c.set_built) tabled.push_back(c.tgc);
      }
    if (!flat_check_) tabled.clear();
    s->flat_slots = 0;
    if (!indexed.empty() && mark_rsetless_slots(&blob, indexed)) {
      s->flat_slots = static_cast<uint32_t>(mark_flat_slots(&blob, tabled));
      if (cudaMemcpyAsync(s->prog.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, stream) != cudaSuccess ||
          cudaStreamSynchronize(stream) != cudaSuccess)
        return std::string("snapshot upload failed: ") + cudaGetErrorString(cudaGetLastError());
    }
    // the range records of the SF_FLAT slots' push step classes, built whole from this layout's rows (a class whose
    // children may reach 0xFFFF has none: record_meet marks its unused lookups with it)
    for (auto& r : s->records) r.rec.release();
    s->records.clear();
    const DSlot* slots = reinterpret_cast<const DSlot*>(blob.data() + ph->off_slots);
    const DUnit* units = reinterpret_cast<const DUnit*>(blob.data() + ph->off_units);
    for (uint32_t sl = 0; flat_records_ && s->flat_slots && sl < ph->n_slots; ++sl) {
      if (!(slots[sl].flags & SF_FLAT)) continue;
      const DUnit& u = units[slots[sl].unit];
      for (int i = u.push_begin; i < u.step_end; ++i) {
        const DStep& st = steps[i];
        bool seen = h.n_objects[h.cls[st.gc].stype] >= 65536u;
        for (const auto& r : s->records) seen = seen || r.gc == st.gc;
        if (seen || s->records.size() == static_cast<size_t>(kMaxFlatRecords)) continue;
        s->records.emplace_back();
        s->records.back().gc = st.gc;
        s->records.back().row_base = st.row_base;
        s->records.back().nres = st.nres;
        s->records.back().ncls = st.ncls;
      }
    }
    build_flat_records(s.get(), nullptr);
  }
  s->revision = revision;

  // occupancy for this program size (dynamic shared memory = program + warp stacks)
  size_t sm = smem_bytes(s->prog_bytes);
  if (sm > 200 * 1024) return "schema program too large for shared memory";
  {
    // The attribute is per function, i.e. shared by every engine of the process (several
    // engines / shards may publish programs of different sizes): only ever raise it.
    static std::mutex attr_mu;
    static size_t attr_by_device[64] = {0};
    size_t& attr_bytes = attr_by_device[device & 63];
    std::lock_guard<std::mutex> g(attr_mu);
    if (sm > attr_bytes) {
      for (auto k : {check_kernel<false>, check_kernel<true>, check_kernel<false, true>, check_kernel<false, false, kMeetNone>,
                     check_kernel<true, false, kMeetNone>, check_kernel<false, true, kMeetNone>, check_kernel<false, false, kMeet16>,
                     check_kernel<true, false, kMeet16>, check_kernel<false, true, kMeet16>,
                     check_kernel<false, false, kMeetSig16>, check_kernel<true, false, kMeetSig16>,
                     check_kernel<false, true, kMeetSig16>, check_kernel<false, false, kMeetSig32>,
                     check_kernel<true, false, kMeetSig32>, check_kernel<false, true, kMeetSig32>,
                     check_kernel<false, false, kMeetSet16>, check_kernel<true, false, kMeetSet16>,
                     check_kernel<false, true, kMeetSet16>, check_kernel<false, false, kMeetSet16, true>,
                     check_kernel<true, false, kMeetSet16, true>})
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sm));
      attr_bytes = sm;
    }
  }
  int occ = 0, occ_c = 0, occ_s = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, check_kernel<false>, kThreads, sm);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_s, check_kernel<false, true>, kThreads, sm);
  if (occ_s < occ) occ = occ_s;  // one grid size serves both
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_c, check_kernel<true>, kThreads, sm);
  if (occ < 1 || occ_c < 1) return "check kernel cannot be resident (occupancy 0)";
  blocks_per_sm_ = occ;
  blocks_per_sm_count_ = occ_c;
  size_t warps = static_cast<size_t>(sm_count_) * std::max(occ, occ_c) * kWarpsPerBlock;
  if (!spill_.ensure(warps * spill_cap_ * sizeof(uint4))) return "out of device memory (spill areas)";
  if (const char* v = std::getenv("ZGPU_MEMO_AFTER")) memo_after_ = static_cast<uint32_t>(std::atoi(v));
  if (!memo_.ensure(warps * memo_entries_ * sizeof(unsigned long long))) memo_entries_ = 0;  // optional
  // readers that already hold the old snapshot keep it alive until they finish
  snap = s;
  return "";
}

int Device::run_pass(const Snapshot& s, const zg_check* queries, uint64_t nq, uint8_t* val, uint8_t* out, bool final_codes,
                     bool raw, zg_check* subq, uint32_t* subq_parent, cudaStream_t st, bool count, std::string* err,
                     const unsigned long long* ready, bool lean) {
  KParams p{};
  p.ready = ready;
  p.row_ptr = s.row_ptr.as<uint32_t>();
  p.col = s.col.as<uint32_t>();
  p.exp = s.exp.p ? s.exp.as<uint32_t>() : nullptr;
  p.rrow_ptr = s.rrow_ptr.as<uint32_t>();
  p.rcol = s.rcol.as<uint32_t>();
  p.invert = (invert && shard_count <= 1) ? 1 : 0;  // a shard does not hold the subject's reverse rows
  p.prog = s.prog.as<uint8_t>();
  p.prog_bytes = s.prog_bytes;
  p.queries = queries;
  p.nq = nq;
  p.L = s.max_leaves;
  p.val = val;
  p.out = out;
  p.final_codes = final_codes;
  unsigned long long* ctrl = ctrl_.as<unsigned long long>();
  p.next = ctrl;
  p.subq_count = ctrl + 1;
  p.alg_bytes = ctrl + 2;
  p.flags = reinterpret_cast<uint32_t*>(ctrl + 3);
  p.events = ctrl + 8;
  p.spill = spill_.as<uint4>();
  p.spill_cap = spill_cap_;
  p.subq = subq;
  p.subq_parent = subq_parent;
  p.subq_cap = subq ? subq_cap_ : 0;
  p.now = now;
  p.budget = budget_;
  p.raw_items = raw;
  p.memo = memo_.as<unsigned long long>();
  p.memo_entries = memo_.p ? memo_entries_ : 0;
  p.memo_after = memo_after_;
  p.shard_count = shard_count;
  p.shard_rank = shard_rank;
  p.no_wildcards = no_wildcards_ ? 1 : 0;
  int meet = s.has_l2 ? kMeet32 : kMeetNone;
  bool all_sig = true, all_set = true;
  for (const auto& c : s.closure)
    if (c.built) {
      p.closure[p.n_closure++] = ClosureRef{c.row_ptr.as<uint32_t>(), c.col.p, c.nsubj, c.tgc, c.width,
                                            c.sig_words ? c.sig.as<unsigned long long>() : nullptr, c.sig_words,
                                            c.set_built ? c.set_hdr.as<unsigned long long>() : nullptr,
                                            c.set_built ? c.set_tab.as<unsigned long long>() : nullptr};
      if (c.width == 2) meet = kMeet16;  // every built index of a snapshot has the same width
      all_sig = all_sig && c.sig_words;
      all_set = all_set && c.set_built;
    }
  for (const auto& r : s.records)
    if (r.built) p.rec[p.n_rec++] = FlatRecordRef{r.rec.as<uint4>(), r.nres, r.gc};
  if (p.n_closure && all_sig && all_set && meet == kMeet16) meet = kMeetSet16;
  else if (p.n_closure && all_sig) meet |= kMeetSig;
  // SF_FLAT slots are marked only where every pair they meet over has signatures and a set table, but another pair
  // may lack them (the snapshot then meets through kMeetSig16): flat_check_kernel runs only with kMeetSet16, whose
  // check_kernel answers its residual. Not for streamed items, which are still landing.
  const bool flat = lean && s.flat_slots && meet == kMeetSet16 && p.invert && !ready && nq < (1ull << 32);
  if (!flat) ZG_CUDA(cudaMemsetAsync(ctrl, 0, 16, st));  // next, subq_count (flat_check_kernel clears them itself)
  const int per_sm = count ? blocks_per_sm_count_ : blocks_per_sm_;
  uint64_t want = (nq + kThreads - 1) / kThreads;
  int grid = static_cast<int>(std::min<uint64_t>(want, static_cast<uint64_t>(sm_count_) * per_sm));
  if (grid < 1) grid = 1;
  size_t sm = smem_bytes(s.prog_bytes);
  // a schema without a two-level step runs the kernel built without the two-level meet; one with 16-bit closure
  // indexes the kernel whose meet reads them; one whose every built index has signatures the kernel that tests them,
  // and one whose every built index also has a set table the kernel that confirms the signatures' "maybe"s in it
  auto pick = [meet](auto none, auto m32, auto m16, auto s32, auto s16, auto t16) {
    return meet == kMeetNone    ? none
           : meet == kMeet16    ? m16
           : meet == kMeetSig16 ? s16
           : meet == kMeetSig32 ? s32
           : meet == kMeetSet16 ? t16
                                : m32;
  };
  if (flat) {
    if (!flat_idx_.ensure(nq * sizeof(uint32_t))) {
      if (err) *err = "out of device memory (residual list)";
      return ZG_ENOMEM;
    }
    p.idx = flat_idx_.as<uint32_t>();
    p.nq_dev = flat_ctrl_.as<unsigned long long>();
    ZG_CUDA(cudaMemsetAsync(p.nq_dev, 0, 8, st));
    const unsigned fgrid = static_cast<unsigned>((nq + kFlatThreads - 1) / kFlatThreads);
    if (count) flat_check_kernel<true><<<fgrid, kFlatThreads, 0, st>>>(p);
    else flat_check_kernel<false><<<fgrid, kFlatThreads, 0, st>>>(p);
    ZG_CUDA(cudaGetLastError());
    ++launches;
    // the residual pass, launched as a programmatic dependent (Hopper): its blocks start as the lean kernel's finish
    // and wait in cudaGridDependencySynchronize for its residual list, instead of after a full launch gap
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = sm;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    ZG_CUDA(count ? cudaLaunchKernelEx(&cfg, check_kernel<true, false, kMeetSet16, true>, p)
                  : cudaLaunchKernelEx(&cfg, check_kernel<false, false, kMeetSet16, true>, p));
    ++launches;
    return ZG_OK;
  }
  if (count)
    pick(check_kernel<true, false, kMeetNone>, check_kernel<true>, check_kernel<true, false, kMeet16>,
         check_kernel<true, false, kMeetSig32>, check_kernel<true, false, kMeetSig16>,
         check_kernel<true, false, kMeetSet16>)<<<grid, kThreads, sm, st>>>(p);
  else if (ready)
    pick(check_kernel<false, true, kMeetNone>, check_kernel<false, true>, check_kernel<false, true, kMeet16>,
         check_kernel<false, true, kMeetSig32>, check_kernel<false, true, kMeetSig16>,
         check_kernel<false, true, kMeetSet16>)<<<grid, kThreads, sm, st>>>(p);
  else
    pick(check_kernel<false, false, kMeetNone>, check_kernel<false>, check_kernel<false, false, kMeet16>,
         check_kernel<false, false, kMeetSig32>, check_kernel<false, false, kMeetSig16>,
         check_kernel<false, false, kMeetSet16>)<<<grid, kThreads, sm, st>>>(p);
  ZG_CUDA(cudaGetLastError());
  ++launches;
  return ZG_OK;
}

uint64_t Device::flat_residual() {
  unsigned long long n[2] = {0, 0};
  // after the last call's kernels, whichever stream the caller enqueued them on
  if (flat_ctrl_.p && cudaSetDevice(device) == cudaSuccess &&
      (!have_last_ || cudaStreamWaitEvent(stream, last_done_, 0) == cudaSuccess) &&
      cudaMemcpyAsync(n, flat_ctrl_.p, sizeof n, cudaMemcpyDeviceToHost, stream) == cudaSuccess)
    cudaStreamSynchronize(stream);
  return n[1];
}

void Device::read_events(uint64_t* spills, uint64_t* memo_batches) {
  unsigned long long ev[2] = {0, 0};
  if (ctrl_.p && cudaSetDevice(device) == cudaSuccess &&
      cudaMemcpyAsync(ev, ctrl_.as<unsigned long long>() + 8, sizeof ev, cudaMemcpyDeviceToHost, stream) == cudaSuccess)
    cudaStreamSynchronize(stream);
  *spills = ev[0];
  *memo_batches = ev[1];
}

int Device::read_phase_clocks(uint64_t* cycles, std::string* err) {
  if (!ZG_PHASE_CLOCKS) {
    if (err) *err = "library built without phase clocks (scripts/build_variant.sh NAME -DZG_PHASE_CLOCKS=1)";
    return ZG_EINVAL;
  }
  unsigned long long ph[kPhases] = {0};
  ZG_CUDA(cudaSetDevice(device));
  ZG_CUDA(cudaMemcpyAsync(ph, ctrl_.as<unsigned long long>() + 11, sizeof ph, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  for (int i = 0; i < kPhases; ++i) cycles[i] = ph[i];
  return ZG_OK;
}

void Device::finish_timing() {
  if (!timing_pending_) return;
  if (cudaEventSynchronize(ev1_) == cudaSuccess) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, ev0_, ev1_) == cudaSuccess) last_ms = ms;
  }
  timing_pending_ = false;
}

int Device::check_device(const zg_check* d_items, uint64_t n, uint8_t* d_out, cudaStream_t st, bool raw_items,
                         uint64_t* count_bytes, std::string* err, bool top, const unsigned long long* ready) {
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published (call zg_publish after loading relationships)";
    return ZG_ENOSNAPSHOT;
  }
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  // st == NULL is the caller's legacy default stream, not the engine's own stream.
  // Scratch (ctrl_, spill_, pass buffers) is shared by every call: order this call
  // after the previous one even when they were enqueued on different streams.
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(st, last_done_, 0));
  const bool count = count_bytes != nullptr;
  unsigned long long* ctrl = ctrl_.as<unsigned long long>();
  // alg_bytes and the sticky flags (spill overflow, budget hit) are cleared once per caller-level
  // call: the halves of a split batch accumulate into them
  if (top) {
    ZG_CUDA(cudaMemsetAsync(ctrl + 2, 0, 16, st));
    cudaEventRecord(ev0_, st);
  }
  const uint32_t L = s->max_leaves;
  int rc = ZG_OK;
  if (!s->has_nonpure) {
    // every slot is a relation or a pure union: one leaf per check, answered in one launch
    rc = run_pass(*s, d_items, n, nullptr, d_out, true, raw_items, nullptr, nullptr, st, count, err, ready, true);
    if (rc) return rc;
  } else {
    if (n * L >= (1ull << 32)) {
      if (err) *err = "batch too large for one call (n * leaves >= 2^32)";
      return ZG_EINVAL;
    }
    std::vector<uint64_t> nq;  // queries per pass level
    auto level = [&](size_t lv) {
      if (q_.size() <= lv) {
        q_.resize(lv + 1);
        parent_.resize(lv + 1);
        val_.resize(lv + 1);
      }
    };
    const zg_check* queries = d_items;
    uint64_t cur = n;
    bool raw = raw_items;
    for (size_t lv = 0; cur > 0; ++lv) {
      if (lv > ZG_MAX_DEPTH + 1) {
        if (err) *err = "sub-query passes exceeded the depth cap";
        return ZG_ECUDA;
      }
      level(lv + 1);
      nq.push_back(cur);
      if (cur * L >= (1ull << 32)) {
        if (err) *err = "pass too large (queries * leaves >= 2^32)";
        return ZG_EINVAL;
      }
      if (!val_[lv].ensure(cur * L + 4) || !q_[lv + 1].ensure(subq_cap_ * sizeof(zg_check)) ||
          !parent_[lv + 1].ensure(subq_cap_ * 4)) {
        if (err) *err = "out of device memory (pass buffers)";
        return ZG_ENOMEM;
      }
      // leaves the kernel skips (short circuit of the boolean tree) must read as "false"
      ZG_CUDA(cudaMemsetAsync(val_[lv].p, 0, cur * L + 4, st));
      // Level 0 writes the v1 codes straight into d_out: when the pass raises no sub-query (the
      // common case: edges into a non-pure permission are rare) they are final and nothing is folded.
      rc = run_pass(*s, queries, cur, val_[lv].as<uint8_t>(), lv == 0 ? d_out : nullptr, true, raw,
                    q_[lv + 1].as<zg_check>(), parent_[lv + 1].as<uint32_t>(), st, count, err, lv == 0 ? ready : nullptr,
                    lv == 0);
      if (rc) return rc;
      unsigned long long host_ctrl[4];
      ZG_CUDA(cudaMemcpyAsync(host_ctrl, ctrl, sizeof host_ctrl, cudaMemcpyDeviceToHost, st));
      ZG_CUDA(cudaStreamSynchronize(st));
      if (host_ctrl[1] > subq_cap_) {
        // more sub-queries than the pass buffer holds: checks are independent, so answer the
        // batch in two halves (each raises about half as many) instead of failing the call
        if (n < 2) {
          if (err) *err = "sub-query buffer overflow on a single check: raise zg_config.subquery_capacity";
          return ZG_ENOMEM;
        }
        const uint64_t half = n / 2;
        ++split_batches;
        int r1 = check_device(d_items, half, d_out, st, raw_items, nullptr, err, false);
        if (r1) return r1;
        return check_device(d_items + half, n - half, d_out + half, st, raw_items, nullptr, err, false);
      }
      cur = host_ctrl[1];
      queries = q_[lv + 1].as<zg_check>();
      raw = false;
      if (cur) ++passes;
    }
    if (nq.size() > 1) {
      for (size_t lv = nq.size(); lv-- > 0;) {
        const unsigned blk = 256;
        const uint64_t m = nq[lv];
        fold_kernel<<<static_cast<unsigned>((m + blk - 1) / blk), blk, 0, st>>>(
            s->prog.as<uint8_t>(), lv == 0 ? d_items : q_[lv].as<zg_check>(), m, L, val_[lv].as<uint8_t>(),
            lv == 0 ? d_out : nullptr, lv == 0 ? nullptr : parent_[lv].as<uint32_t>(),
            lv == 0 ? nullptr : val_[lv - 1].as<uint8_t>(), 0);
        ++launches;
      }
      ZG_CUDA(cudaGetLastError());
    }
  }
  if (top) {
    cudaEventRecord(ev1_, st);
    timing_pending_ = true;
  }
  cudaEventRecord(last_done_, st);
  have_last_ = true;
  checks += n;
  if (count) {
    unsigned long long host_ctrl[4];
    ZG_CUDA(cudaMemcpyAsync(host_ctrl, ctrl, sizeof host_ctrl, cudaMemcpyDeviceToHost, st));
    ZG_CUDA(cudaStreamSynchronize(st));
    *count_bytes = host_ctrl[2];
    last_alg_bytes = host_ctrl[2];
  }
  return ZG_OK;
}

int Device::check_host(const zg_check* items, uint64_t n, uint8_t* out, std::string* err) {
  std::vector<HostReq> one{{items, n, out}};
  return check_host_multi(one, err);
}

// One launch sequence for the requests of one or several callers (see Batcher in capi.cu).
//
// Host buffers -> answers, copies included. Large inputs are STREAMED: the items go up in chunks on a copy
// stream, each chunk followed by an 8-byte copy of "items landed so far" into the word the kernel polls, and
// the check kernel -- launched once, persistent -- starts on the first chunk while the rest is still on the
// PCIe bus (warps wait for their batch: KParams::ready). H2D and the kernel overlap without per-chunk
// launches, whose tails cost more than the copies (DESIGN.md 4, "tried and reverted").
int Device::check_host_multi(const std::vector<HostReq>& reqs, std::string* err) {
  uint64_t total = 0;
  for (const auto& r : reqs) total += r.n;
  if (total == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (!stage_in_.ensure(total * sizeof(zg_check)) || !stage_out_.ensure(total)) {
    if (err) *err = "out of device memory (staging)";
    return ZG_ENOMEM;
  }
  // Pinned caller buffers (zg_host_alloc) are copied straight from/to; pageable ones and the requests of
  // several callers go through the engine's pinned staging area.
  cudaPointerAttributes a{};
  const bool single = reqs.size() == 1;
  const bool in_pinned = single && cudaPointerGetAttributes(&a, reqs[0].items) == cudaSuccess && a.type == cudaMemoryTypeHost;
  const bool out_pinned = single && cudaPointerGetAttributes(&a, reqs[0].out) == cudaSuccess && a.type == cudaMemoryTypeHost;
  cudaGetLastError();
  if (!in_pinned && pin_in_cap_ < total * sizeof(zg_check)) {
    if (pin_in_) cudaFreeHost(pin_in_);
    pin_in_cap_ = 0;
    ZG_CUDA(cudaMallocHost(&pin_in_, total * sizeof(zg_check)));
    pin_in_cap_ = total * sizeof(zg_check);
  }
  if (!out_pinned && pin_out_cap_ < total) {
    if (pin_out_) cudaFreeHost(pin_out_);
    pin_out_cap_ = 0;
    ZG_CUDA(cudaMallocHost(&pin_out_, total));
    pin_out_cap_ = total;
  }
  unsigned long long* d_ready = ctrl_.as<unsigned long long>() + 10;
  const bool streamed = total >= kStreamMinItems;
  const unsigned long long* ready_arg = nullptr;
  // A large group of many callers (1 000 lists of 10 000 items under BASELINE config 5): one thread gathering 16 B per
  // item into the staging area takes longer than the kernel that answers them. Helpers copy contiguous shares.
  bool gathered = false;
  if (!in_pinned && total >= kParallelGatherItems && reqs.size() >= 2 * kGatherThreads) {
    std::vector<uint64_t> start(reqs.size() + 1, 0);
    for (size_t i = 0; i < reqs.size(); ++i) start[i + 1] = start[i] + reqs[i].n;
    auto share = [&](unsigned t) {
      const size_t b = reqs.size() * t / kGatherThreads, e = reqs.size() * (t + 1) / kGatherThreads;
      for (size_t i = b; i < e; ++i)
        std::memcpy(static_cast<zg_check*>(pin_in_) + start[i], reqs[i].items, reqs[i].n * sizeof(zg_check));
    };
    std::thread helpers[kGatherThreads - 1];
    for (unsigned t = 1; t < kGatherThreads; ++t) helpers[t - 1] = std::thread(share, t);
    share(0);
    for (auto& h : helpers) h.join();
    gathered = true;
  }
  if (!streamed) {
    const void* src = reqs[0].items;
    if (gathered) {
      src = pin_in_;
    } else if (!in_pinned) {
      uint64_t off = 0;
      for (const auto& r : reqs) {
        std::memcpy(static_cast<zg_check*>(pin_in_) + off, r.items, r.n * sizeof(zg_check));
        off += r.n;
      }
      src = pin_in_;
    }
    ZG_CUDA(cudaMemcpyAsync(stage_in_.p, src, total * sizeof(zg_check), cudaMemcpyHostToDevice, stream));
  } else {
    // copy stream: after the previous call (it may still read stage_in_ / the ready word), reset the word,
    // then chunk, count, chunk, count ... ; the compute stream only waits for the reset
    const uint64_t n_chunks = (total + kStreamChunkItems - 1) / kStreamChunkItems;
    if (pin_ready_cap_ < n_chunks) {
      if (pin_ready_) cudaFreeHost(pin_ready_);
      pin_ready_cap_ = 0;
      ZG_CUDA(cudaMallocHost(&pin_ready_, n_chunks * 8));
      pin_ready_cap_ = n_chunks;
    }
    if (have_last_) ZG_CUDA(cudaStreamWaitEvent(cstream_, last_done_, 0));
    ZG_CUDA(cudaMemsetAsync(d_ready, 0, 8, cstream_));
    ZG_CUDA(cudaEventRecord(ev_reset_, cstream_));
    ZG_CUDA(cudaStreamWaitEvent(stream, ev_reset_, 0));
    size_t ri = 0;          // request being gathered
    uint64_t roff = 0;      // items of it already gathered
    for (uint64_t ck = 0; ck < n_chunks; ++ck) {
      const uint64_t b = ck * kStreamChunkItems, e = std::min(total, b + kStreamChunkItems);
      const zg_check* src;
      if (in_pinned) {
        src = reqs[0].items + b;
      } else if (gathered) {
        src = static_cast<const zg_check*>(pin_in_) + b;
      } else {
        zg_check* dst = static_cast<zg_check*>(pin_in_) + b;
        uint64_t need = e - b, w = 0;
        while (need) {
          const uint64_t take = std::min(need, reqs[ri].n - roff);
          std::memcpy(dst + w, reqs[ri].items + roff, take * sizeof(zg_check));
          w += take;
          roff += take;
          need -= take;
          if (roff == reqs[ri].n) {
            ++ri;
            roff = 0;
          }
        }
        src = dst;
      }
      ZG_CUDA(cudaMemcpyAsync(stage_in_.as<zg_check>() + b, src, (e - b) * sizeof(zg_check), cudaMemcpyHostToDevice, cstream_));
      pin_ready_[ck] = e;
      ZG_CUDA(cudaMemcpyAsync(d_ready, pin_ready_ + ck, 8, cudaMemcpyHostToDevice, cstream_));
    }
    ready_arg = d_ready;
    ++streamed_calls;
  }
  int rc = check_device(stage_in_.as<zg_check>(), total, stage_out_.as<uint8_t>(), stream, true, nullptr, err, true, ready_arg);
  if (rc) {
    if (streamed) cudaStreamSynchronize(cstream_);  // nothing of this call may still be in flight
    return rc;
  }
  void* dst = out_pinned ? static_cast<void*>(reqs[0].out) : pin_out_;
  ZG_CUDA(cudaMemcpyAsync(dst, stage_out_.p, total, cudaMemcpyDeviceToHost, stream));
  uint32_t flags = 0;
  ZG_CUDA(cudaMemcpyAsync(&flags, ctrl_.as<unsigned long long>() + 3, 4, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  if (streamed) ZG_CUDA(cudaStreamSynchronize(cstream_));
  if (flags & 32u) {
    if (err) *err = "host-to-device copy of the request stalled (streamed admission timed out)";
    return ZG_ECUDA;
  }
  if (flags & 1u) {
    if (err) *err = "expansion stack overflow (per-warp spill area exhausted)";
    return ZG_ENOMEM;
  }
  if (!out_pinned) {
    uint64_t off = 0;
    for (const auto& r : reqs) {
      std::memcpy(r.out, static_cast<uint8_t*>(pin_out_) + off, r.n);
      off += r.n;
    }
  }
  if (!single) {
    ++coalesced_launches;
    coalesced_requests += reqs.size();
  }
  return ZG_OK;
}

// ---- sharded store: one pass per call; the raised sub-queries are exchanged device to device -------------------

int Device::route_by_owner(const zg_check* d_items, uint64_t n, int level, uint32_t n_dest, zg_check* d_routed, uint32_t* d_src,
                           uint64_t* counts, std::string* err) {
  if (n_dest == 0 || n_dest > kMaxRouteDest) {
    if (err) *err = "route_by_owner: destination count out of range";
    return ZG_EINVAL;
  }
  for (uint32_t d = 0; d < n_dest; ++d) counts[d] = 0;
  ZG_CUDA(cudaSetDevice(device));
  if (!d_items) {
    const size_t lv = static_cast<size_t>(level);
    if (lv >= shard_nsub_.size() || n != shard_nsub_[lv]) {
      if (err) *err = "route_by_owner: level / count mismatch";
      return ZG_EINVAL;
    }
    d_items = q_[lv + 1].as<zg_check>();
  }
  return route_<true>(d_items, n, n_dest, ResOwner{}, d_routed, d_src, counts, err);
}

// Counting sort of n items by owner(item, n_dest) into d_routed (destination-major), with their source indices in
// d_src when kSrc; counts[d] (host) = items for destination d.
template <bool kSrc, class Item, class Owner>
int Device::route_(const Item* d_items, uint64_t n, uint32_t n_dest, Owner owner, Item* d_routed, uint32_t* d_src, uint64_t* counts,
                   std::string* err) {
  if (n_dest == 0 || n_dest > kMaxRouteDest) {  // the histogram and the cursors hold kMaxRouteDest destinations
    if (err) *err = "routing: destination count out of range (1 .. 64)";
    return ZG_EINVAL;
  }
  for (uint32_t d = 0; d < n_dest; ++d) counts[d] = 0;
  if (n == 0) return ZG_OK;
  if (!route_ctrl_.ensure(2 * kMaxRouteDest * 8)) return ZG_ENOMEM;
  unsigned long long* d_counts = route_ctrl_.as<unsigned long long>();
  unsigned long long* d_cursor = d_counts + kMaxRouteDest;
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  ZG_CUDA(cudaMemsetAsync(d_counts, 0, kMaxRouteDest * 8, stream));
  const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + 255) / 256, static_cast<uint64_t>(sm_count_) * 8));
  route_count_kernel<<<grid, 256, 0, stream>>>(d_items, n, n_dest, d_counts, owner);
  unsigned long long h[kMaxRouteDest];
  ZG_CUDA(cudaMemcpyAsync(h, d_counts, n_dest * 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  unsigned long long off[kMaxRouteDest], acc = 0;
  for (uint32_t d = 0; d < n_dest; ++d) {
    counts[d] = h[d];
    off[d] = acc;
    acc += h[d];
  }
  ZG_CUDA(cudaMemcpyAsync(d_cursor, off, n_dest * 8, cudaMemcpyHostToDevice, stream));
  route_scatter_kernel<Item, Owner, kSrc><<<grid, 256, 0, stream>>>(d_items, n, n_dest, d_cursor, d_routed, d_src, owner);
  launches += 2;
  ZG_CUDA(cudaGetLastError());
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  return ZG_OK;
}

// Buffers per level lv: q_[lv] = this level's queries (stage_in_ at level 0), val_[lv] = their leaf values,
// q_[lv+1] / parent_[lv+1] = the sub-queries the pass raised (the same buffers the single-GPU multi-pass loop
// uses; here their consumers live on other ranks).
int Device::shard_pass_dev(const zg_check* d_queries, uint64_t n, int level, uint64_t* n_sub, std::string* err) {
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  ZG_CUDA(cudaSetDevice(device));
  const size_t lv = static_cast<size_t>(level);
  if (q_.size() <= lv + 1) {
    q_.resize(lv + 2);
    parent_.resize(lv + 2);
    val_.resize(lv + 2);
  }
  if (shard_nq_.size() <= lv) {
    shard_nq_.resize(lv + 1);
    shard_nsub_.resize(lv + 1);
  }
  shard_nq_[lv] = n;
  shard_nsub_[lv] = 0;
  *n_sub = 0;
  if (n == 0) return ZG_OK;
  const uint32_t L = s->max_leaves;
  if (n * L >= (1ull << 32)) {
    if (err) *err = "pass too large (n * leaves >= 2^32)";
    return ZG_EINVAL;
  }
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  // the level's queries are kept (the fold re-reads them): own copy, device to device
  DevBuf& qbuf = lv == 0 ? stage_in_ : q_[lv];
  if (!qbuf.ensure(std::max<size_t>(n * sizeof(zg_check), lv == 0 ? 0 : subq_cap_ * sizeof(zg_check))) ||
      !val_[lv].ensure(n * L + 4) || !q_[lv + 1].ensure(subq_cap_ * sizeof(zg_check)) || !parent_[lv + 1].ensure(subq_cap_ * 4)) {
    if (err) *err = "out of device memory (shard pass buffers)";
    return ZG_ENOMEM;
  }
  ZG_CUDA(cudaMemcpyAsync(qbuf.p, d_queries, n * sizeof(zg_check), cudaMemcpyDeviceToDevice, stream));
  unsigned long long* ctrl = ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 2, 0, 16, stream));
  ZG_CUDA(cudaMemsetAsync(val_[lv].p, 0, n * L + 4, stream));
  // level 0 items come from callers (flags ignored); deeper levels are raised sub-queries (flags = hop depth)
  int rc = run_pass(*s, qbuf.as<zg_check>(), n, val_[lv].as<uint8_t>(), nullptr, false, level == 0, q_[lv + 1].as<zg_check>(),
                    parent_[lv + 1].as<uint32_t>(), stream, false, err);
  if (rc) return rc;
  unsigned long long host_ctrl[4];
  ZG_CUDA(cudaMemcpyAsync(host_ctrl, ctrl, sizeof host_ctrl, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  const uint32_t flags = static_cast<uint32_t>(host_ctrl[3] & 0xFFFFFFFFu);
  if (host_ctrl[1] > subq_cap_) {
    if (err) *err = "sub-query buffer overflow: raise zg_config.subquery_capacity or shrink the batch";
    return ZG_ENOMEM;
  }
  if (flags & 1u) {
    if (err) *err = "expansion stack overflow";
    return ZG_ENOMEM;
  }
  shard_nsub_[lv] = host_ctrl[1];
  *n_sub = host_ctrl[1];
  checks += level == 0 ? n : 0;
  ++passes;
  return ZG_OK;
}

int Device::shard_fold_dev(int level, const uint8_t* d_child_vals, const uint32_t* d_src, uint64_t n_sub, uint8_t* d_out,
                           bool final_codes, std::string* err) {
  std::shared_ptr<Snapshot> s = snap;
  const size_t lv = static_cast<size_t>(level);
  if (!s || lv >= shard_nq_.size() || n_sub != shard_nsub_[lv]) {
    if (err) *err = "shard_fold_dev: level / count mismatch";
    return ZG_EINVAL;
  }
  const uint64_t n = shard_nq_[lv];
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  const unsigned blk = 256;
  if (n_sub) {
    or_children_src_kernel<<<static_cast<unsigned>((n_sub + blk - 1) / blk), blk, 0, stream>>>(
        parent_[lv + 1].as<uint32_t>(), d_src, d_child_vals, n_sub, val_[lv].as<uint8_t>());
    ++launches;
  }
  const DevBuf& qbuf = lv == 0 ? stage_in_ : q_[lv];
  fold_kernel<<<static_cast<unsigned>((n + blk - 1) / blk), blk, 0, stream>>>(
      s->prog.as<uint8_t>(), qbuf.as<zg_check>(), n, s->max_leaves, val_[lv].as<uint8_t>(), d_out, nullptr, nullptr,
      final_codes ? 0 : 1);
  ++launches;
  ZG_CUDA(cudaGetLastError());
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  return ZG_OK;
}

int Device::unroute(const uint32_t* d_src, const uint8_t* d_val, uint64_t n, uint8_t* d_out, std::string* err) {
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unroute_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(d_src, d_val, n, d_out);
  ++launches;
  ZG_CUDA(cudaGetLastError());
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  return ZG_OK;
}

// ---- sharded handle (capi.cu run_sharded): the levels of DeviceShardedChecker, exchanged through peer memory --------
static_assert(kMaxShards == kMaxRouteDest, "a PeerTable holds every routing destination");

int Device::peer_events_(std::string* err) {
  if (!ev_peer_[0])
    for (cudaEvent_t& ev : ev_peer_) ZG_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  return ZG_OK;
}

int Device::peer_begin(const zg_check* items, uint64_t n, uint64_t* counts, std::string* err) {
  for (uint32_t d = 0; d < own_count; ++d) counts[d] = 0;
  home_n_ = n;
  ZG_CUDA(cudaSetDevice(device));
  if (int rc = peer_events_(err)) return rc;
  if (!pin_peer_) ZG_CUDA(cudaMallocHost(&pin_peer_, (4 + kMaxShards) * sizeof(unsigned long long)));
  if (!peer_ctrl_.ensure(2 * kMaxShards * sizeof(unsigned long long)) || !home_.ensure(n * sizeof(zg_check)) ||
      !home_pos_.ensure(n * 4) || !home_out_.ensure(n)) {
    if (err) *err = "out of device memory (sharded handle buffers)";
    return ZG_ENOMEM;
  }
  if (n == 0) return ZG_OK;
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* d_counts = peer_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemcpyAsync(home_.p, items, n * sizeof(zg_check), cudaMemcpyDefault, stream));
  ZG_CUDA(cudaMemsetAsync(d_counts, 0, kMaxShards * sizeof(unsigned long long), stream));
  const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + 255) / 256, static_cast<uint64_t>(sm_count_) * 8));
  route_count_kernel<<<grid, 256, 0, stream>>>(home_.as<zg_check>(), n, own_count, d_counts);
  ZG_CUDA(cudaGetLastError());
  ++launches;
  ZG_CUDA(cudaMemcpyAsync(pin_peer_, d_counts, own_count * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  for (uint32_t d = 0; d < own_count; ++d) counts[d] = pin_peer_[d];
  return ZG_OK;
}

zg_check* Device::peer_inbox(int level, uint64_t n, std::string* err) {
  const size_t lv = static_cast<size_t>(level);
  if (pl_.size() <= lv) pl_.resize(lv + 1);
  PeerLevel& L = pl_[lv];
  L.nq = n;
  L.nsub = 0;
  if (cudaSetDevice(device) != cudaSuccess || !L.in.ensure(std::max<uint64_t>(n, 1) * sizeof(zg_check))) {
    if (err) *err = "out of device memory (sharded handle inbox)";
    return nullptr;
  }
  return L.in.as<zg_check>();
}

int Device::peer_scatter(int level, const PeerTable& t, std::string* err) {
  const bool callers = level == 0;
  const PeerLevel* from = callers ? nullptr : &pl_[static_cast<size_t>(level) - 1];
  const uint64_t n = callers ? home_n_ : from->nsub;
  ZG_CUDA(cudaSetDevice(device));
  if (n) {
    unsigned long long* d_cursor = peer_ctrl_.as<unsigned long long>() + kMaxShards;
    ZG_CUDA(cudaMemsetAsync(d_cursor, 0, kMaxShards * sizeof(unsigned long long), stream));
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + 255) / 256, static_cast<uint64_t>(sm_count_) * 8));
    peer_scatter_kernel<<<grid, 256, 0, stream>>>(callers ? home_.as<zg_check>() : from->raised.as<zg_check>(), n, own_count,
                                                  d_cursor, t, callers ? home_pos_.as<uint32_t>() : from->pos.as<uint32_t>());
    ZG_CUDA(cudaGetLastError());
    ++launches;
  }
  ZG_CUDA(cudaEventRecord(peer_event(level), stream));
  return ZG_OK;
}

int Device::peer_pass(int level, const std::vector<cudaEvent_t>& wait, uint64_t* n_sub, uint64_t* counts, bool* overflow,
                      bool no_wildcards, std::string* err) {
  for (uint32_t d = 0; d < own_count; ++d) counts[d] = 0;
  *n_sub = 0;
  *overflow = false;
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  PeerLevel& L = pl_[static_cast<size_t>(level)];
  if (L.nq == 0) return ZG_OK;
  const uint64_t nq = L.nq, Lv = s->max_leaves;
  if (nq * Lv >= (1ull << 32)) {
    if (err) *err = "pass too large (queries * leaves >= 2^32)";
    return ZG_EINVAL;
  }
  ZG_CUDA(cudaSetDevice(device));
  for (cudaEvent_t ev : wait) ZG_CUDA(cudaStreamWaitEvent(stream, ev, 0));
  if (!L.val.ensure(nq * Lv + 4) || !L.out.ensure(nq) || !L.raised.ensure(subq_cap_ * sizeof(zg_check)) ||
      !L.parent.ensure(subq_cap_ * 4) || !L.pos.ensure(subq_cap_ * 4)) {
    if (err) *err = "out of device memory (sharded handle pass buffers)";
    return ZG_ENOMEM;
  }
  unsigned long long* ctrl = ctrl_.as<unsigned long long>();
  unsigned long long* d_counts = peer_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 2, 0, 16, stream));
  ZG_CUDA(cudaMemsetAsync(L.val.p, 0, nq * Lv + 4, stream));
  // level 0: the callers' items (flags ignored), v1 codes written straight out (final unless the level raised
  // sub-queries: then peer_fold rewrites them); deeper: routed sub-queries (flags = hop depth), value bits
  no_wildcards_ = no_wildcards;
  int rc = run_pass(*s, L.in.as<zg_check>(), nq, L.val.as<uint8_t>(), L.out.as<uint8_t>(), level == 0, level == 0,
                    L.raised.as<zg_check>(), L.parent.as<uint32_t>(), stream, false, err);
  no_wildcards_ = false;
  if (rc) return rc;
  ZG_CUDA(cudaMemsetAsync(d_counts, 0, kMaxShards * sizeof(unsigned long long), stream));
  const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(subq_cap_ / 256 + 1, static_cast<uint64_t>(sm_count_) * 8));
  peer_count_kernel<<<grid, 256, 0, stream>>>(L.raised.as<zg_check>(), ctrl + 1, subq_cap_, own_count, d_counts);
  ZG_CUDA(cudaGetLastError());
  ++launches;
  ZG_CUDA(cudaMemcpyAsync(pin_peer_, ctrl, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(pin_peer_ + 4, d_counts, own_count * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  const uint64_t raised = pin_peer_[1];
  const uint32_t flags = static_cast<uint32_t>(pin_peer_[3] & 0xFFFFFFFFu);
  *n_sub = raised;
  if (raised > subq_cap_) {
    *overflow = true;
    return ZG_OK;
  }
  if (flags & 1u) {
    if (err) *err = "expansion stack overflow (per-warp spill area exhausted)";
    return ZG_ENOMEM;
  }
  L.nsub = raised;
  for (uint32_t d = 0; d < own_count; ++d) counts[d] = pin_peer_[4 + d];
  if (level == 0) checks += nq;
  else ++passes;
  return ZG_OK;
}

int Device::peer_fold(int level, const PeerTable& t, const std::vector<cudaEvent_t>& wait, std::string* err) {
  const PeerLevel& L = pl_[static_cast<size_t>(level)];
  if (L.nsub == 0) return ZG_OK;  // the pass's own values are final
  std::shared_ptr<Snapshot> s = snap;
  ZG_CUDA(cudaSetDevice(device));
  for (cudaEvent_t ev : wait) ZG_CUDA(cudaStreamWaitEvent(stream, ev, 0));
  const unsigned blk = 256;
  peer_or_children_kernel<<<static_cast<unsigned>((L.nsub + blk - 1) / blk), blk, 0, stream>>>(
      L.raised.as<zg_check>(), L.parent.as<uint32_t>(), L.pos.as<uint32_t>(), L.nsub, own_count, t, L.val.as<uint8_t>());
  fold_kernel<<<static_cast<unsigned>((L.nq + blk - 1) / blk), blk, 0, stream>>>(
      s->prog.as<uint8_t>(), L.in.as<zg_check>(), L.nq, s->max_leaves, L.val.as<uint8_t>(), L.out.as<uint8_t>(), nullptr,
      nullptr, level == 0 ? 0 : 1);
  ZG_CUDA(cudaGetLastError());
  launches += 2;
  ZG_CUDA(cudaEventRecord(peer_event(level), stream));
  return ZG_OK;
}

int Device::peer_finish(const PeerTable& t, const std::vector<cudaEvent_t>& wait, uint8_t* out, std::string* err) {
  ZG_CUDA(cudaSetDevice(device));
  if (home_n_) {
    for (cudaEvent_t ev : wait) ZG_CUDA(cudaStreamWaitEvent(stream, ev, 0));
    peer_gather_kernel<<<static_cast<unsigned>((home_n_ + 255) / 256), 256, 0, stream>>>(
        home_.as<zg_check>(), home_pos_.as<uint32_t>(), home_n_, own_count, t, home_out_.as<uint8_t>());
    ZG_CUDA(cudaGetLastError());
    ++launches;
    ZG_CUDA(cudaMemcpyAsync(out, home_out_.p, home_n_, cudaMemcpyDefault, stream));
  }
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  return ZG_OK;
}

bool Device::hl_ensure(DevBuf& b, uint64_t bytes) { return cudaSetDevice(device) == cudaSuccess && b.ensure(std::max<uint64_t>(bytes, 8)); }

int Device::peer_put(const unsigned long long* src, uint64_t n, uint32_t n_dest, const PeerTable& t, int level, std::string* err) {
  ZG_CUDA(cudaSetDevice(device));
  if (int rc = peer_events_(err)) return rc;
  if (n) {
    if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + 255) / 256, static_cast<uint64_t>(sm_count_) * 8));
    peer_put_kernel<<<grid, 256, 0, stream>>>(src, n, n_dest, t);
    ZG_CUDA(cudaGetLastError());
    ++launches;
  }
  ZG_CUDA(cudaEventRecord(peer_event(level), stream));
  return ZG_OK;
}

int Device::peer_wait(const std::vector<cudaEvent_t>& wait, std::string* err) {
  ZG_CUDA(cudaSetDevice(device));
  for (cudaEvent_t ev : wait) ZG_CUDA(cudaStreamWaitEvent(stream, ev, 0));
  return ZG_OK;
}

// ---- LookupResources on the object-hash sharded store (DESIGN.md 4, dist.DeviceShardedLookup) ------------------
// sl_ctrl_ words: [0] flags, [1] candidates, [2] keys, [3] error mask, then the level counts, then first[] / end[] of
// every lookup's answers after the final sort.
namespace {
constexpr size_t kSlCounts = 8, kSlFirst = kSlCounts + ZG_MAX_DEPTH + 4, kSlEnd = kSlFirst + kMaxLookupBatch,
                 kSlCtrlWords = kSlEnd + kMaxLookupBatch;
}

int Device::shard_lookup_begin(const std::vector<LookupReq>& reqs, const uint8_t* home, uint64_t walk_cap,
                               unsigned long long* d_seeds, std::string* err) {
  std::shared_ptr<Snapshot> s = snap;
  const size_t K = reqs.size();
  sl_snap_.reset();
  ss_snap_.reset();  // a sharded LookupSubjects round shares the walk buffers
  sl_n_cand_ = sl_n_walk_ = 0;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  if (K == 0 || K > kMaxLookupBatch || walk_cap == 0 || shard_count > kMaxRouteDest) {
    if (err) *err = "shard_lookup_begin: 1..64 lookups, a non-zero walk capacity and at most 64 shards";
    return ZG_EINVAL;
  }
  for (size_t k = 0; k < K; ++k)
    if (reqs[k].res_type >= s->n_objects.size() || reqs[k].proto.stype >= s->n_objects.size() || home[k] >= shard_count) {
      if (err) *err = "shard_lookup_begin: unknown type or home rank";
      return ZG_EINVAL;
    }
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  const unsigned long long words = (s->total_bits + 31) / 32 + 4;
  if (!rb_visited_.ensure(words * 4 * K) || !lk_jobs_.ensure((walk_cap + K) * sizeof(zg_check)) || !lb_owner_.ensure(walk_cap + K) ||
      !lb_params_.ensure(K * sizeof(LookupParam)) || !sl_home_.ensure(K) || !sl_ctrl_.ensure(kSlCtrlWords * 8)) {
    if (err) *err = "out of device memory (sharded lookup buffers)";
    return ZG_ENOMEM;
  }
  std::vector<LookupParam> lp(K);
  std::vector<unsigned long long> seeds(K);
  for (size_t i = 0; i < K; ++i) {
    const zg_check& q = reqs[i].proto;
    lp[i] = LookupParam{q.subj, reqs[i].res_type, q.perm, q.stype, q.srel};
    seeds[i] = (static_cast<unsigned long long>(i) << 48) | (static_cast<unsigned long long>(q.stype) << 32) | q.subj;
  }
  ZG_CUDA(cudaMemsetAsync(sl_ctrl_.p, 0, kSlCtrlWords * 8, stream));
  ZG_CUDA(cudaMemsetAsync(rb_visited_.p, 0, words * 4 * K, stream));
  ZG_CUDA(cudaMemcpyAsync(lb_params_.p, lp.data(), K * sizeof(LookupParam), cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemcpyAsync(sl_home_.p, home, K, cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemcpyAsync(d_seeds, seeds.data(), K * 8, cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  sl_snap_ = s;
  sl_reqs_ = reqs;
  sl_cap_ = walk_cap;
  return ZG_OK;
}

int Device::shard_lookup_expand(const unsigned long long* d_front, uint64_t n_in, int level, unsigned long long* d_next,
                                uint64_t* n_next, bool* overflow, std::string* err) {
  *n_next = 0;
  *overflow = false;
  if (!sl_snap_ || level < 0 || level > ZG_MAX_DEPTH + 1) {
    if (err) *err = "shard_lookup_expand: no round begun, or level out of range";
    return ZG_EINVAL;
  }
  // the gathered frontier is the same on every rank, so every rank reports this overflow in the same level
  if (n_in > sl_cap_) {
    *overflow = true;
    return ZG_OK;
  }
  if (n_in == 0) return ZG_OK;
  const Snapshot& s = *sl_snap_;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* ctrl = sl_ctrl_.as<unsigned long long>();
  unsigned long long* counts = ctrl + kSlCounts;
  const unsigned long long c[2] = {n_in, 0};
  ZG_CUDA(cudaMemcpyAsync(counts + level, c, sizeof c, cudaMemcpyHostToDevice, stream));
  MrbfsParams p{};
  p.rrow_ptr = s.rrow_ptr.as<uint32_t>();
  p.rcol = s.rcol.as<uint32_t>();
  p.prog = s.prog.as<uint8_t>();
  p.lk = lb_params_.as<LookupParam>();
  p.in = d_front;
  p.out = d_next;
  p.counts = counts;
  p.level = level;
  p.cap = sl_cap_;
  p.visited = rb_visited_.as<uint32_t>();
  p.words = (s.total_bits + 31) / 32 + 4;
  p.type_bit_base = s.type_bit_base.as<unsigned long long>();
  p.cand = lk_jobs_.as<zg_check>();
  p.cand_owner = lb_owner_.as<uint8_t>();
  p.cand_count = ctrl + 1;
  p.cand_cap = sl_cap_;
  p.flags = reinterpret_cast<uint32_t*>(ctrl);
  mrbfs_expand_kernel<<<sm_count_ * 8, 256, 0, stream>>>(p);
  ++launches;
  ZG_CUDA(cudaGetLastError());
  unsigned long long flags = 0, cnt = 0;
  ZG_CUDA(cudaMemcpyAsync(&flags, ctrl, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(&cnt, counts + level + 1, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  *overflow = (static_cast<uint32_t>(flags) & 16u) != 0;
  *n_next = std::min<uint64_t>(cnt, sl_cap_);
  return ZG_OK;
}

int Device::shard_lookup_candidates(bool exhaustive, zg_check* d_items, uint64_t cap, uint64_t* n, std::string* err) {
  *n = 0;
  if (!sl_snap_) {
    if (err) *err = "shard_lookup_candidates: no round begun";
    return ZG_EINVAL;
  }
  Snapshot& s = *sl_snap_;
  const size_t K = sl_reqs_.size();
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* ctrl = sl_ctrl_.as<unsigned long long>();
  const unsigned long long words = (s.total_bits + 31) / 32 + 4;
  // userset subjects T:x#r of lookups of type T whose x this shard owns: x is a member of T:x#P for every relation r
  // inlined into P, and the walk only reaches x through stored edges (run_lookup_group asks the check kernel the same)
  std::vector<SelfCand> self;
  uint64_t bit_base = 0;
  for (size_t k = 0; k < K; ++k) {
    const LookupReq& r = sl_reqs_[k];
    const zg_check& q = r.proto;
    if (q.srel == kNone || q.stype != r.res_type || q.subj >= ZG_NO_OBJECT - 1 || q.subj % shard_count != shard_rank) continue;
    bit_base = 0;
    for (uint16_t t = 0; t < r.res_type; ++t) bit_base += (uint64_t(s.n_objects[t]) + 31) & ~31ull;
    self.push_back(SelfCand{static_cast<uint32_t>(k), 0, q.subj < s.n_objects[r.res_type] ? bit_base + q.subj : ~0ull});
  }
  uint64_t need = self.size();
  unsigned long long walked = 0;
  if (exhaustive) {
    if (s.resources_stale) {
      std::string rerr = gpu_resource_lists(&s, stream);
      if (!rerr.empty()) {
        if (err) *err = rerr;
        return ZG_ECUDA;
      }
    }
    for (const LookupReq& r : sl_reqs_) need += s.n_resources[r.res_type];
  } else {
    ZG_CUDA(cudaMemcpyAsync(&walked, ctrl + 1, 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if (walked > sl_cap_) {
      if (err) *err = "shard_lookup_candidates: the walk overflowed (redo the round in halves, or exhaustive)";
      return ZG_EINVAL;
    }
    need += walked;
  }
  if (!d_items) {
    *n = need;
    return ZG_OK;
  }
  if (cap < need) {
    if (err) *err = "shard_lookup_candidates: item buffer too small";
    return ZG_E2BIG;
  }
  if (exhaustive) {
    if (!lk_jobs_.ensure(std::max<uint64_t>(need, 1) * sizeof(zg_check)) || !lb_owner_.ensure(std::max<uint64_t>(need, 1))) {
      if (err) *err = "out of device memory (sharded lookup candidates)";
      return ZG_ENOMEM;
    }
    ZG_CUDA(cudaMemsetAsync(rb_visited_.p, 0, words * 4 * K, stream));
    uint64_t at = 0;
    for (size_t k = 0; k < K; ++k) {
      const LookupReq& r = sl_reqs_[k];
      const uint64_t nr = s.n_resources[r.res_type];
      if (!nr) continue;
      uint64_t base = 0;
      for (uint16_t t = 0; t < r.res_type; ++t) base += (uint64_t(s.n_objects[t]) + 31) & ~31ull;
      const LookupParam l{r.proto.subj, r.res_type, r.proto.perm, r.proto.stype, r.proto.srel};
      lookup_fill_owned_kernel<<<static_cast<unsigned>((nr + 255) / 256), 256, 0, stream>>>(
          s.resources[r.res_type].as<uint32_t>(), nr, l, static_cast<uint32_t>(k), rb_visited_.as<uint32_t>() + k * words, base,
          lk_jobs_.as<zg_check>() + at, lb_owner_.as<uint8_t>() + at);
      ++launches;
      at += nr;
    }
    const unsigned long long filled = at;
    ZG_CUDA(cudaMemcpyAsync(ctrl + 1, &filled, 8, cudaMemcpyHostToDevice, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));  // `filled` lives on this stack frame
  }
  // the self-membership candidates come after these: only the walk's / the fill's can fail the lookup
  sl_n_walk_ = exhaustive ? need - self.size() : walked;
  if (!self.empty()) {
    if (!sl_self_.ensure(self.size() * sizeof(SelfCand))) return ZG_ENOMEM;
    ZG_CUDA(cudaMemcpyAsync(sl_self_.p, self.data(), self.size() * sizeof(SelfCand), cudaMemcpyHostToDevice, stream));
    lookup_self_kernel<<<1, kMaxLookupBatch, 0, stream>>>(lb_params_.as<LookupParam>(), sl_self_.as<SelfCand>(),
                                                          static_cast<uint32_t>(self.size()), rb_visited_.as<uint32_t>(), words,
                                                          lk_jobs_.as<zg_check>(), lb_owner_.as<uint8_t>(), ctrl + 1);
    ++launches;
  }
  unsigned long long total = 0;
  ZG_CUDA(cudaMemcpyAsync(&total, ctrl + 1, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  if (total) ZG_CUDA(cudaMemcpyAsync(d_items, lk_jobs_.p, total * sizeof(zg_check), cudaMemcpyDeviceToDevice, stream));
  ZG_CUDA(cudaGetLastError());
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  sl_n_cand_ = total;
  *n = total;
  return ZG_OK;
}

int Device::shard_lookup_route(const uint8_t* d_codes, uint64_t n, uint32_t n_dest, unsigned long long* d_routed,
                               uint64_t* counts, std::string* err) {
  for (uint32_t d = 0; d < n_dest && d < kMaxRouteDest; ++d) counts[d] = 0;
  if (!sl_snap_ || n != sl_n_cand_ || n_dest != shard_count) {
    if (err) *err = "shard_lookup_route: no candidates of this round, or a count / shard count mismatch";
    return ZG_EINVAL;
  }
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  if (!lb_keys_[0].ensure(n * 8)) {
    if (err) *err = "out of device memory (sharded lookup keys)";
    return ZG_ENOMEM;
  }
  unsigned long long* ctrl = sl_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 2, 0, 16, stream));
  // per-lookup counts of this shard's answers are not needed: the home rank counts after the final sort
  lookup_keys_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
      lk_jobs_.as<zg_check>(), lb_owner_.as<uint8_t>(), d_codes, n, lb_keys_[0].as<unsigned long long>(), ctrl + 2,
      ctrl + kSlFirst, ctrl + 3, sl_n_walk_);
  ++launches;
  unsigned long long n_keys = 0;
  ZG_CUDA(cudaMemcpyAsync(&n_keys, ctrl + 2, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  have_last_ = true;
  return route_<false>(static_cast<const unsigned long long*>(lb_keys_[0].as<unsigned long long>()), n_keys, n_dest,
                       KeyHomeOwner{sl_home_.as<uint8_t>()}, d_routed, static_cast<uint32_t*>(nullptr), counts, err);
}

int Device::shard_lookup_finish(const unsigned long long* d_keys, uint64_t n, uint32_t* d_ids, uint64_t* per_lookup,
                                uint64_t* err_mask, std::string* err) {
  *err_mask = 0;
  if (!sl_snap_) {
    if (err) *err = "shard_lookup_finish: no round begun";
    return ZG_EINVAL;
  }
  const size_t K = sl_reqs_.size();
  // the round ends here, whatever follows: the snapshot it read is not kept resident past it
  sl_snap_.reset();
  sl_reqs_.clear();
  sl_n_cand_ = sl_n_walk_ = 0;
  for (size_t k = 0; k < K; ++k) per_lookup[k] = 0;
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  if (!lb_keys_[1].ensure(n * 8)) {
    if (err) *err = "out of device memory (sharded lookup keys)";
    return ZG_ENOMEM;
  }
  unsigned long long* ctrl = sl_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 3, 0, 8, stream));
  ZG_CUDA(cudaMemsetAsync(ctrl + kSlFirst, 0, 2 * kMaxLookupBatch * 8, stream));
  // ascending (error bit, lookup, id): answers per lookup in lookup order, the error keys last
  std::string serr = sort_u64(d_keys, lb_keys_[1].as<unsigned long long>(), n, kErrKeyBit + 1, stream);
  if (!serr.empty()) {
    if (err) *err = serr;
    return ZG_ECUDA;
  }
  lookup_split_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
      lb_keys_[1].as<unsigned long long>(), n, d_ids, ctrl + kSlFirst, ctrl + kSlEnd, ctrl + 3);
  ++launches;
  unsigned long long host[1 + 2 * kMaxLookupBatch];
  ZG_CUDA(cudaMemcpyAsync(host, ctrl + 3, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(host + 1, ctrl + kSlFirst, 2 * kMaxLookupBatch * 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaGetLastError());
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  *err_mask = host[0];
  for (size_t k = 0; k < K; ++k) per_lookup[k] = host[1 + kMaxLookupBatch + k] - host[1 + k];
  return ZG_OK;
}

int Device::shard_pass_nowild_dev(const zg_check* d_queries, uint64_t n, int level, uint64_t* n_sub, std::string* err) {
  no_wildcards_ = true;
  const int rc = shard_pass_dev(d_queries, n, level, n_sub, err);
  no_wildcards_ = false;
  return rc;
}

// ---- LookupSubjects on the object-hash sharded store (DESIGN.md 4, dist.DeviceShardedLookup.lookup_subjects) -------
// ss_ctrl_ words: [0] flags, [1] outbox entries, [2] admitted entries, [3] candidates, [4] keys, [5] no-wildcards
// items, [6] granted mask, [7] failed mask, then first[] / end[] of the 128 answer runs after the final sort.
namespace {
constexpr size_t kSsFirst = 8, kSsEnd = kSsFirst + 2 * kMaxLookupBatch, kSsCtrlWords = kSsEnd + 2 * kMaxLookupBatch;

SsWalkParams ss_walk_params(const Snapshot& s, const SubjectsParam* lk, uint32_t* visited, unsigned long long* ctrl, uint32_t rank,
                            uint32_t count) {
  SsWalkParams p{};
  p.row_ptr = s.row_ptr.as<uint32_t>();
  p.col = s.col.as<uint32_t>();
  p.fwd = s.ls_fwd.as<FwdClass>();
  p.type_off = s.ls_type_off.as<uint32_t>();
  p.mask = s.ls_mask.as<uint32_t>();
  p.mask_words = s.ls_mask_words;
  p.shard_rank = rank;
  p.shard_count = count;
  p.lk = lk;
  p.visited = visited;
  p.words = (s.total_bits + 31) / 32 + 4;
  p.type_bit_base = s.type_bit_base.as<unsigned long long>();
  p.flags = reinterpret_cast<uint32_t*>(ctrl);
  return p;
}
}  // namespace

int Device::shard_subjects_begin(const std::vector<SubjectsReq>& reqs, const uint8_t* home, uint64_t include, uint64_t walk_cap,
                                 unsigned long long* d_front, uint64_t* n_front, std::string* err) {
  std::shared_ptr<Snapshot> s = snap;
  const size_t K = reqs.size();
  *n_front = 0;
  ss_snap_.reset();
  sl_snap_.reset();  // a sharded LookupResources round shares the walk buffers
  ss_n_cand_ = ss_n_nw_ = 0;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  if (K == 0 || K > kMaxLookupBatch || walk_cap == 0 || shard_count > kMaxRouteDest) {
    if (err) *err = "shard_subjects_begin: 1..64 lookups, a non-zero walk capacity and at most 64 shards";
    return ZG_EINVAL;
  }
  for (size_t k = 0; k < K; ++k)
    if (reqs[k].res_type >= s->n_objects.size() || reqs[k].stype >= s->n_objects.size() || home[k] >= shard_count) {
      if (err) *err = "shard_subjects_begin: unknown type or home rank";
      return ZG_EINVAL;
    }
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  const unsigned long long words = (s->total_bits + 31) / 32 + 4;
  if (!rb_visited_.ensure(words * 4 * K) || !lk_jobs_.ensure((walk_cap + K) * sizeof(zg_check)) || !lb_owner_.ensure(walk_cap + K) ||
      !lb_params_.ensure(K * sizeof(SubjectsParam)) || !ss_out_.ensure(std::max<uint64_t>(walk_cap, K) * 8) || !ss_home_.ensure(K) ||
      !ss_ctrl_.ensure(kSsCtrlWords * 8)) {
    if (err) *err = "out of device memory (sharded lookup buffers)";
    return ZG_ENOMEM;
  }
  std::vector<SubjectsParam> lp(K);
  std::vector<unsigned long long> seeds;
  ss_probes_.clear();
  ss_probe_owner_.clear();
  for (size_t k = 0; k < K; ++k) {
    const SubjectsReq& r = reqs[k];
    lp[k] = SubjectsParam{r.res, r.res_type, r.perm, r.stype, r.srel};
    // a resource no relationship names has an empty answer (n_objects is the same on every shard)
    if (r.res >= s->n_objects[r.res_type] || r.res % shard_count != shard_rank) continue;
    zg_check q{};
    q.res = r.res;
    q.subj = ZG_NO_OBJECT - 1;
    q.perm = r.perm;
    q.stype = r.stype;
    q.srel = r.srel;
    ss_probes_.push_back(q);
    ss_probe_owner_.push_back(static_cast<uint8_t>(k));
    seeds.push_back((static_cast<unsigned long long>(k) << 48) | (static_cast<unsigned long long>(r.res_type) << 32) | r.res);
  }
  const unsigned long long n_probe = ss_probes_.size();
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl, 0, kSsCtrlWords * 8, stream));
  ZG_CUDA(cudaMemsetAsync(rb_visited_.p, 0, words * 4 * K, stream));
  ZG_CUDA(cudaMemcpyAsync(lb_params_.p, lp.data(), K * sizeof(SubjectsParam), cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemcpyAsync(ss_home_.p, home, K, cudaMemcpyHostToDevice, stream));
  if (n_probe) {
    ZG_CUDA(cudaMemcpyAsync(lk_jobs_.p, ss_probes_.data(), n_probe * sizeof(zg_check), cudaMemcpyHostToDevice, stream));
    ZG_CUDA(cudaMemcpyAsync(lb_owner_.p, ss_probe_owner_.data(), n_probe, cudaMemcpyHostToDevice, stream));
    ZG_CUDA(cudaMemcpyAsync(ctrl + 3, &n_probe, 8, cudaMemcpyHostToDevice, stream));
    ZG_CUDA(cudaMemcpyAsync(ss_out_.p, seeds.data(), seeds.size() * 8, cudaMemcpyHostToDevice, stream));
  }
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));  // the host arrays above live on this frame
  ss_snap_ = s;
  ss_reqs_ = reqs;
  ss_cap_ = walk_cap;
  ss_include_ = include;
  // the seeds are admitted like any arrived entry: a resource of the subject type becomes its own candidate
  return shard_subjects_admit(ss_out_.as<unsigned long long>(), seeds.size(), d_front, n_front, err);
}

int Device::shard_subjects_expand(const unsigned long long* d_front, uint64_t n_in, uint32_t n_dest, unsigned long long* d_routed,
                                  uint64_t* counts, bool* overflow, std::string* err) {
  *overflow = false;
  for (uint32_t d = 0; d < n_dest && d < kMaxRouteDest; ++d) counts[d] = 0;
  if (!ss_snap_ || n_dest != shard_count || n_in > ss_cap_) {
    if (err) *err = "shard_subjects_expand: no round begun, a shard count mismatch, or a frontier over the walk capacity";
    return ZG_EINVAL;
  }
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 1, 0, 8, stream));
  if (n_in) {
    SsWalkParams p = ss_walk_params(*ss_snap_, lb_params_.as<SubjectsParam>(), rb_visited_.as<uint32_t>(), ctrl, shard_rank, shard_count);
    p.in = d_front;
    p.n_in = n_in;
    p.out = ss_out_.as<unsigned long long>();
    p.out_count = ctrl + 1;
    p.cap = ss_cap_;
    ss_expand_kernel<<<sm_count_ * 8, 256, 0, stream>>>(p);
    ++launches;
    ZG_CUDA(cudaGetLastError());
  }
  unsigned long long host[2] = {0, 0};
  ZG_CUDA(cudaMemcpyAsync(host, ctrl, sizeof host, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  // flags are sticky: an admission (or the begin's) that did not fit is reported here
  *overflow = (static_cast<uint32_t>(host[0]) & 16u) != 0;
  if (*overflow) return ZG_OK;
  return route_<false>(static_cast<const unsigned long long*>(ss_out_.as<unsigned long long>()), host[1], n_dest, EntryOwner{},
                       d_routed, static_cast<uint32_t*>(nullptr), counts, err);
}

int Device::shard_subjects_expand_count(const unsigned long long* d_front, uint64_t n_in, uint64_t* counts, bool* overflow,
                                        std::string* err) {
  *overflow = false;
  for (uint32_t d = 0; d < shard_count && d < kMaxRouteDest; ++d) counts[d] = 0;
  if (!ss_snap_ || shard_count > kMaxRouteDest || n_in > ss_cap_) {
    if (err) *err = "shard_subjects_expand_count: no round begun, or a frontier over the walk capacity";
    return ZG_EINVAL;
  }
  ZG_CUDA(cudaSetDevice(device));
  if (int rc = peer_events_(err)) return rc;
  if (!pin_peer_) ZG_CUDA(cudaMallocHost(&pin_peer_, (4 + kMaxShards) * sizeof(unsigned long long)));
  if (!peer_ctrl_.ensure(2 * kMaxShards * sizeof(unsigned long long))) {
    if (err) *err = "out of device memory (sharded handle buffers)";
    return ZG_ENOMEM;
  }
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  unsigned long long* d_counts = peer_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 1, 0, 8, stream));
  ZG_CUDA(cudaMemsetAsync(d_counts, 0, kMaxShards * sizeof(unsigned long long), stream));
  if (n_in) {
    SsWalkParams p = ss_walk_params(*ss_snap_, lb_params_.as<SubjectsParam>(), rb_visited_.as<uint32_t>(), ctrl, shard_rank, shard_count);
    p.in = d_front;
    p.n_in = n_in;
    p.out = ss_out_.as<unsigned long long>();
    p.out_count = ctrl + 1;
    p.cap = ss_cap_;
    ss_expand_kernel<<<sm_count_ * 8, 256, 0, stream>>>(p);
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>(ss_cap_ / 256 + 1, static_cast<uint64_t>(sm_count_) * 8));
    peer_entry_count_kernel<<<grid, 256, 0, stream>>>(ss_out_.as<unsigned long long>(), ctrl + 1, ss_cap_, shard_count, d_counts);
    launches += 2;
    ZG_CUDA(cudaGetLastError());
  }
  ZG_CUDA(cudaMemcpyAsync(pin_peer_, ctrl, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(pin_peer_ + 4, d_counts, shard_count * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  // flags are sticky: an admission (or the begin's) that did not fit is reported here
  *overflow = (static_cast<uint32_t>(pin_peer_[0]) & 16u) != 0;
  if (*overflow) return ZG_OK;
  for (uint32_t d = 0; d < shard_count; ++d) counts[d] = pin_peer_[4 + d];
  return ZG_OK;
}

int Device::shard_subjects_scatter(uint64_t n, const PeerTable& t, int level, std::string* err) {
  if (!ss_snap_ || n > ss_cap_) {
    if (err) *err = "shard_subjects_scatter: no round begun, or an outbox over the walk capacity";
    return ZG_EINVAL;
  }
  ZG_CUDA(cudaSetDevice(device));
  if (n) {
    unsigned long long* d_cursor = peer_ctrl_.as<unsigned long long>() + kMaxShards;
    ZG_CUDA(cudaMemsetAsync(d_cursor, 0, kMaxShards * sizeof(unsigned long long), stream));
    const unsigned grid = static_cast<unsigned>(std::min<uint64_t>((n + 255) / 256, static_cast<uint64_t>(sm_count_) * 8));
    peer_entry_scatter_kernel<<<grid, 256, 0, stream>>>(ss_out_.as<unsigned long long>(), n, shard_count, d_cursor, t);
    ZG_CUDA(cudaGetLastError());
    ++launches;
  }
  ZG_CUDA(cudaEventRecord(peer_event(level), stream));
  return ZG_OK;
}

int Device::shard_subjects_admit(const unsigned long long* d_in, uint64_t n_in, unsigned long long* d_next, uint64_t* n_next,
                                 std::string* err) {
  *n_next = 0;
  if (!ss_snap_) {
    if (err) *err = "shard_subjects_admit: no round begun";
    return ZG_EINVAL;
  }
  if (n_in == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 2, 0, 8, stream));
  SsWalkParams p = ss_walk_params(*ss_snap_, lb_params_.as<SubjectsParam>(), rb_visited_.as<uint32_t>(), ctrl, shard_rank, shard_count);
  p.in = d_in;
  p.n_in = n_in;
  p.out = d_next;
  p.out_count = ctrl + 2;
  p.cap = ss_cap_;
  p.cand = lk_jobs_.as<zg_check>();
  p.cand_owner = lb_owner_.as<uint8_t>();
  p.cand_count = ctrl + 3;
  p.cand_cap = ss_cap_ + ss_probes_.size();
  ss_admit_kernel<<<static_cast<unsigned>((n_in + 255) / 256), 256, 0, stream>>>(p);
  ++launches;
  ZG_CUDA(cudaGetLastError());
  unsigned long long cnt = 0;
  ZG_CUDA(cudaMemcpyAsync(&cnt, ctrl + 2, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  *n_next = std::min<uint64_t>(cnt, ss_cap_);
  return ZG_OK;
}

int Device::shard_subjects_candidates(bool exhaustive, zg_check* d_items, uint64_t cap, uint64_t* n, std::string* err) {
  *n = 0;
  if (!ss_snap_) {
    if (err) *err = "shard_subjects_candidates: no round begun";
    return ZG_EINVAL;
  }
  const Snapshot& s = *ss_snap_;
  const size_t K = ss_reqs_.size();
  const uint64_t n_probe = ss_probes_.size();
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  std::vector<uint64_t> owned(K, 0);  // exhaustive: ids rank, rank + shard_count, ... below n_objects of the subject type
  unsigned long long need = n_probe;
  if (exhaustive) {
    for (size_t k = 0; k < K; ++k) {
      const uint64_t no = s.n_objects[ss_reqs_[k].stype];
      owned[k] = no > shard_rank ? (no - shard_rank - 1) / shard_count + 1 : 0;
      need += owned[k];
    }
  } else {
    ZG_CUDA(cudaMemcpyAsync(&need, ctrl + 3, 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if (need > ss_cap_ + n_probe) {
      if (err) *err = "shard_subjects_candidates: the walk overflowed (redo the round in halves, or exhaustive)";
      return ZG_EINVAL;
    }
  }
  if (!d_items) {
    *n = need;
    return ZG_OK;
  }
  if (cap < need) {
    if (err) *err = "shard_subjects_candidates: item buffer too small";
    return ZG_E2BIG;
  }
  if (exhaustive) {
    if (!lk_jobs_.ensure(std::max<uint64_t>(need, 1) * sizeof(zg_check)) || !lb_owner_.ensure(std::max<uint64_t>(need, 1))) {
      if (err) *err = "out of device memory (sharded lookup candidates)";
      return ZG_ENOMEM;
    }
    // the probes first (a grown buffer does not keep them), then every owned id of each lookup's subject type
    if (n_probe) {
      ZG_CUDA(cudaMemcpyAsync(lk_jobs_.p, ss_probes_.data(), n_probe * sizeof(zg_check), cudaMemcpyHostToDevice, stream));
      ZG_CUDA(cudaMemcpyAsync(lb_owner_.p, ss_probe_owner_.data(), n_probe, cudaMemcpyHostToDevice, stream));
    }
    uint64_t at = n_probe;
    for (size_t k = 0; k < K; ++k) {
      if (!owned[k]) continue;
      const SubjectsReq& r = ss_reqs_[k];
      ss_fill_owned_kernel<<<static_cast<unsigned>((owned[k] + 255) / 256), 256, 0, stream>>>(
          SubjectsParam{r.res, r.res_type, r.perm, r.stype, r.srel}, static_cast<uint32_t>(k), owned[k], shard_rank, shard_count,
          lk_jobs_.as<zg_check>() + at, lb_owner_.as<uint8_t>() + at);
      ++launches;
      at += owned[k];
    }
    ZG_CUDA(cudaGetLastError());
  }
  if (need) ZG_CUDA(cudaMemcpyAsync(d_items, lk_jobs_.p, need * sizeof(zg_check), cudaMemcpyDeviceToDevice, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  ss_n_cand_ = need;
  *n = need;
  return ZG_OK;
}

int Device::shard_subjects_verdicts(const uint8_t* d_codes, uint64_t n, uint64_t* granted, uint64_t* failed, std::string* err) {
  *granted = *failed = 0;
  if (!ss_snap_ || n != ss_n_cand_) {
    if (err) *err = "shard_subjects_verdicts: no candidates of this round, or a count mismatch";
    return ZG_EINVAL;
  }
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 6, 0, 16, stream));
  ss_verdict_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(lk_jobs_.as<zg_check>(), lb_owner_.as<uint8_t>(), d_codes,
                                                                                n, ctrl + 6, ctrl + 7);
  ++launches;
  ZG_CUDA(cudaGetLastError());
  unsigned long long host[2] = {0, 0};
  ZG_CUDA(cudaMemcpyAsync(host, ctrl + 6, sizeof host, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  *granted = host[0];
  *failed = host[1];
  return ZG_OK;
}

int Device::shard_subjects_nowild(const uint8_t* d_codes, uint64_t n, uint64_t granted, uint64_t failed, zg_check* d_items,
                                  uint64_t cap, uint64_t* n_nw, std::string* err) {
  *n_nw = 0;
  if (!ss_snap_ || n != ss_n_cand_) {
    if (err) *err = "shard_subjects_nowild: no candidates of this round, or a count mismatch";
    return ZG_EINVAL;
  }
  if (cap < n) {
    if (err) *err = "shard_subjects_nowild: item buffer smaller than the candidates";
    return ZG_E2BIG;
  }
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  // every candidate gives at most one key, or one no-wildcards item that gives at most one key
  const uint64_t m = std::max<uint64_t>(n, 1);
  if (!lb_keys_[0].ensure(m * 8) || !ss_nw_.ensure(m * sizeof(zg_check)) || !ss_nw_owner_.ensure(m)) {
    if (err) *err = "out of device memory (sharded lookup keys)";
    return ZG_ENOMEM;
  }
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + 4, 0, 16, stream));
  unsigned long long nw = 0;
  if (n) {
    ss_keys_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
        lk_jobs_.as<zg_check>(), lb_owner_.as<uint8_t>(), d_codes, n, granted, failed, ss_include_, lb_keys_[0].as<unsigned long long>(),
        ctrl + 4, ss_nw_.as<zg_check>(), ss_nw_owner_.as<uint8_t>(), ctrl + 5);
    ++launches;
    ZG_CUDA(cudaGetLastError());
    ZG_CUDA(cudaMemcpyAsync(&nw, ctrl + 5, 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if (nw) ZG_CUDA(cudaMemcpyAsync(d_items, ss_nw_.p, nw * sizeof(zg_check), cudaMemcpyDeviceToDevice, stream));
  }
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  ss_n_nw_ = nw;
  *n_nw = nw;
  return ZG_OK;
}

int Device::shard_subjects_route(const uint8_t* d_codes, uint64_t n, uint32_t n_dest, unsigned long long* d_routed, uint64_t* counts,
                                 std::string* err) {
  for (uint32_t d = 0; d < n_dest && d < kMaxRouteDest; ++d) counts[d] = 0;
  if (!ss_snap_ || n != ss_n_nw_ || n_dest != shard_count) {
    if (err) *err = "shard_subjects_route: no no-wildcards items of this round, or a count / shard count mismatch";
    return ZG_EINVAL;
  }
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  if (n) {
    // granted = failed = 0: each item that checks HAS without the wildcard relationships is listed
    ss_keys_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(
        ss_nw_.as<zg_check>(), ss_nw_owner_.as<uint8_t>(), d_codes, n, 0, 0, 0, lb_keys_[0].as<unsigned long long>(), ctrl + 4,
        nullptr, nullptr, ctrl + 5);
    ++launches;
    ZG_CUDA(cudaGetLastError());
  }
  unsigned long long n_keys = 0;
  ZG_CUDA(cudaMemcpyAsync(&n_keys, ctrl + 4, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  return route_<false>(static_cast<const unsigned long long*>(lb_keys_[0].as<unsigned long long>()), n_keys, n_dest,
                       KeyHomeOwner{ss_home_.as<uint8_t>()}, d_routed, static_cast<uint32_t*>(nullptr), counts, err);
}

int Device::shard_subjects_finish(const unsigned long long* d_keys, uint64_t n, uint32_t* d_ids, uint64_t* listed, uint64_t* excluded,
                                  std::string* err) {
  if (!ss_snap_) {
    if (err) *err = "shard_subjects_finish: no round begun";
    return ZG_EINVAL;
  }
  const size_t K = ss_reqs_.size();
  // the round ends here, whatever follows: the snapshot it read is not kept resident past it
  ss_snap_.reset();
  ss_reqs_.clear();
  ss_n_cand_ = ss_n_nw_ = 0;
  for (size_t k = 0; k < K; ++k) listed[k] = excluded[k] = 0;
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  if (!lb_keys_[1].ensure(n * 8)) {
    if (err) *err = "out of device memory (sharded lookup keys)";
    return ZG_ENOMEM;
  }
  unsigned long long* ctrl = ss_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(ctrl + kSsFirst, 0, 4 * kMaxLookupBatch * 8, stream));
  // ascending (excluded bit, lookup, id): the listed runs in lookup order, then the excluded runs
  std::string serr = sort_u64(d_keys, lb_keys_[1].as<unsigned long long>(), n, kExclKeyBit + 1, stream);
  if (!serr.empty()) {
    if (err) *err = serr;
    return ZG_ECUDA;
  }
  ss_split_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(lb_keys_[1].as<unsigned long long>(), n, d_ids,
                                                                              ctrl + kSsFirst, ctrl + kSsEnd);
  ++launches;
  unsigned long long host[4 * kMaxLookupBatch];
  ZG_CUDA(cudaMemcpyAsync(host, ctrl + kSsFirst, sizeof host, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaGetLastError());
  ZG_CUDA(cudaEventRecord(last_done_, stream));
  have_last_ = true;
  ZG_CUDA(cudaStreamSynchronize(stream));
  const unsigned long long* first = host;
  const unsigned long long* end = host + 2 * kMaxLookupBatch;
  for (size_t k = 0; k < K; ++k) {
    listed[k] = end[k] - first[k];
    excluded[k] = end[kMaxLookupBatch + k] - first[kMaxLookupBatch + k];
  }
  return ZG_OK;
}

int Device::lookup_candidates(const Snapshot& s, uint16_t res_type, const zg_check& proto, uint64_t* n_cand, bool* overflow,
                              std::string* err) {
  *overflow = false;
  *n_cand = 0;
  const size_t vis_bytes = static_cast<size_t>((s.total_bits + 31) / 32) * 4 + 16;
  if (!rb_visited_.ensure(vis_bytes) || !rb_front_[0].ensure(rb_cap_ * 8) || !rb_front_[1].ensure(rb_cap_ * 8) ||
      !rb_cand_.ensure(rb_cap_ * 4)) {
    *overflow = true;  // not enough memory for the BFS buffers: exhaustive scan instead
    return ZG_OK;
  }
  unsigned long long* ctrl = ctrl_.as<unsigned long long>();  // [4] next_count, [5] cand_count; flags at ctrl+3
  ZG_CUDA(cudaMemsetAsync(rb_visited_.p, 0, vis_bytes, stream));
  ZG_CUDA(cudaMemsetAsync(ctrl + 3, 0, 24, stream));
  const unsigned long long seed = (static_cast<unsigned long long>(proto.stype) << 32) | proto.subj;
  ZG_CUDA(cudaMemcpyAsync(rb_front_[0].p, &seed, 8, cudaMemcpyHostToDevice, stream));
  RbfsParams p{};
  p.rrow_ptr = s.rrow_ptr.as<uint32_t>();
  p.rcol = s.rcol.as<uint32_t>();
  p.prog = s.prog.as<uint8_t>();
  p.visited = rb_visited_.as<uint32_t>();
  p.type_bit_base = s.type_bit_base.as<unsigned long long>();
  p.want_type = res_type;
  p.cand = rb_cand_.as<uint32_t>();
  p.cand_count = ctrl + 5;
  p.cand_cap = rb_cap_;
  p.next_count = ctrl + 4;
  p.next_cap = rb_cap_;
  p.flags = reinterpret_cast<uint32_t*>(ctrl + 3);
  unsigned long long n_in = 1;
  int cur = 0;
  for (int level = 0; n_in > 0; ++level) {
    if (level > ZG_MAX_DEPTH + 1) break;  // deeper objects cannot be within the dispatch cap anyway
    p.frontier = rb_front_[cur].as<unsigned long long>();
    p.n_in = n_in;
    p.next = rb_front_[cur ^ 1].as<unsigned long long>();
    p.wildcard_level = (level == 0 && proto.srel == kNone) ? 1 : 0;
    ZG_CUDA(cudaMemsetAsync(ctrl + 4, 0, 8, stream));
    const unsigned blk = 256;
    const unsigned long long threads = n_in * 32;
    rbfs_expand_kernel<<<static_cast<unsigned>((threads + blk - 1) / blk), blk, 0, stream>>>(p);
    ++launches;
    unsigned long long host[3];
    ZG_CUDA(cudaMemcpyAsync(host, ctrl + 3, sizeof host, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if (static_cast<uint32_t>(host[0]) & 16u) {
      *overflow = true;
      return ZG_OK;
    }
    n_in = host[1];
    *n_cand = host[2];
    cur ^= 1;
  }
  return ZG_OK;
}

int Device::lookup(uint16_t res_type, const zg_check& proto, std::vector<uint32_t>* ids, std::string* err) {
  ids->clear();
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  if (res_type >= s->resources.size()) {
    if (err) *err = "unknown resource type";
    return ZG_EINVAL;
  }
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  // flat union of direct relations and a relation-less subject: the answer is the union of
  // the subject's reverse rows (classes of other subject types contribute nothing)
  if (use_rbfs && proto.srel == kNone && proto.perm < s->flat_n.size() && s->flat_n[proto.perm] >= 0) {
    const int nc = s->flat_n[proto.perm];
    const uint64_t cap = rb_cap_;
    if (!rb_cand_.ensure(cap * 4 + 8)) return ZG_ENOMEM;
    // layout: [count u64][ids ...] so the count and the first ids come back in ONE copy
    unsigned long long* d_count = rb_cand_.as<unsigned long long>();
    uint32_t* d_ids = rb_cand_.as<uint32_t>() + 2;
    lookup_flat_kernel<<<1, 32, 0, stream>>>(s->rrow_ptr.as<uint32_t>(), s->rcol.as<uint32_t>(),
                                             s->flat_cls[proto.perm].as<FlatLookupClass>(), nc, proto.stype, proto.subj,
                                             d_ids, cap, d_count);
    ++launches;
    constexpr uint64_t kFirst = 4094;
    static thread_local std::vector<uint32_t> host;
    host.resize(2 + kFirst);
    ZG_CUDA(cudaMemcpyAsync(host.data(), rb_cand_.p, host.size() * 4, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    unsigned long long cnt = 0;
    std::memcpy(&cnt, host.data(), 8);
    if (cnt <= cap) {
      ++lookups_flat;
      ids->resize(cnt);
      const uint64_t first = std::min<uint64_t>(cnt, kFirst);
      if (first) std::memcpy(ids->data(), host.data() + 2, first * 4);
      if (cnt > first) {
        ZG_CUDA(cudaMemcpyAsync(ids->data() + first, d_ids + first, (cnt - first) * 4, cudaMemcpyDeviceToHost, stream));
        ZG_CUDA(cudaStreamSynchronize(stream));
      }
      std::sort(ids->begin(), ids->end());
      ids->erase(std::unique(ids->begin(), ids->end()), ids->end());
      return ZG_OK;
    }
    // more results than the buffer: fall through to the general path
  }
  // candidates: reverse BFS from the subject (superset of the answer), else every resource of the type
  if (s->resources_stale) {
    std::string rerr = gpu_resource_lists(s.get(), stream);
    if (!rerr.empty()) {
      if (err) *err = rerr;
      return ZG_ECUDA;
    }
  }
  uint64_t n = s->n_resources[res_type];
  const uint32_t* cand = s->resources[res_type].as<uint32_t>();
  if (n == 0) return ZG_OK;
  if (use_rbfs && proto.stype < s->n_objects.size()) {
    uint64_t nc = 0;
    bool overflow = false;
    int rc = lookup_candidates(*s, res_type, proto, &nc, &overflow, err);
    if (rc) return rc;
    if (!overflow) {
      ++lookups_rbfs;
      n = nc;
      cand = rb_cand_.as<uint32_t>();
      if (n == 0) return ZG_OK;
    } else {
      ++lookups_exhaustive;
    }
  } else {
    ++lookups_exhaustive;
  }
  const size_t count_off = (n * 4 + 7) & ~size_t(7);  // the result count lives after the ids
  if (!lk_jobs_.ensure(n * sizeof(zg_check)) || !lk_codes_.ensure(n) || !lk_ids_.ensure(count_off + 8)) {
    if (err) *err = "out of device memory (lookup)";
    return ZG_ENOMEM;
  }
  const unsigned blk = 256, grid = static_cast<unsigned>((n + blk - 1) / blk);
  lookup_fill_kernel<<<grid, blk, 0, stream>>>(cand, n, proto, lk_jobs_.as<zg_check>());
  ++launches;
  int rc = check_device(lk_jobs_.as<zg_check>(), n, lk_codes_.as<uint8_t>(), stream, true, nullptr, err);
  if (rc) return rc;
  unsigned long long* d_count = reinterpret_cast<unsigned long long*>(lk_ids_.as<uint8_t>() + count_off);
  ZG_CUDA(cudaMemsetAsync(d_count, 0, 8, stream));
  lookup_compact_kernel<<<grid, blk, 0, stream>>>(cand, lk_codes_.as<uint8_t>(), n, lk_ids_.as<uint32_t>(), n, d_count,
                                                  reinterpret_cast<uint32_t*>(ctrl_.as<unsigned long long>() + 3));
  ++launches;
  unsigned long long cnt = 0;
  uint32_t lflags = 0;
  ZG_CUDA(cudaMemcpyAsync(&cnt, d_count, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(&lflags, ctrl_.as<unsigned long long>() + 3, 4, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  if (lflags & 1u) {
    if (err) *err = "expansion stack overflow (per-warp spill area exhausted)";
    return ZG_ENOMEM;
  }
  if (lflags & 8u) {
    // a candidate's check ended in an error (dispatch depth or work budget): the embedded SpiceDB fails
    // the LookupResources call in that case; a silently shortened answer would read as "not allowed"
    if (err) *err = "LookupResources: a candidate could not be decided (max dispatch depth / work budget exceeded)";
    return ZG_EDEPTH;
  }
  ids->resize(cnt);
  if (cnt) {
    // ascending ids: radix-sort on the device when the answer is large (a host sort of 50 k ids
    // costs milliseconds), into the job buffer that is free again by now
    const uint32_t* src = lk_ids_.as<uint32_t>();
    if (cnt > 2048) {
      std::string serr = sort_u32(lk_ids_.as<uint32_t>(), lk_jobs_.as<uint32_t>(), cnt, stream);
      if (!serr.empty()) {
        if (err) *err = serr;
        return ZG_ECUDA;
      }
      src = lk_jobs_.as<uint32_t>();
    }
    ZG_CUDA(cudaMemcpyAsync(ids->data(), src, cnt * 4, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if (cnt <= 2048) std::sort(ids->begin(), ids->end());
  }
  return ZG_OK;
}

int Device::lookup_page(uint16_t res_type, const zg_check& proto, bool has_after, uint32_t after, uint64_t want, uint32_t self,
                        std::vector<uint32_t>* ids, LookupPageStats* st, std::string* err) {
  ids->clear();
  *st = LookupPageStats{};
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  if (res_type >= s->resources.size()) {
    if (err) *err = "unknown resource type";
    return ZG_EINVAL;
  }
  if (want == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  if (!lp_ctrl_.ensure(4 * 8)) {
    if (err) *err = "out of device memory (lookup page)";
    return ZG_ENOMEM;
  }
  unsigned long long* ctrl = lp_ctrl_.as<unsigned long long>();  // [0] selected / found, [1] self seen / error, [2] bound
  unsigned long long h[3] = {0, 0, 0};
  ZG_CUDA(cudaMemsetAsync(ctrl, 0, 4 * 8, stream));
  // ---- the candidates: those of lookup()
  const uint32_t* cand = nullptr;
  uint64_t n = 0;
  bool flat = false, sorted = false;
  if (use_rbfs && proto.srel == kNone && proto.perm < s->flat_n.size() && s->flat_n[proto.perm] >= 0) {
    const uint64_t cap = rb_cap_;
    if (!rb_cand_.ensure(cap * 4 + 8)) return ZG_ENOMEM;
    unsigned long long* d_count = rb_cand_.as<unsigned long long>();  // as in lookup(): [count u64][ids ...]
    lookup_flat_kernel<<<1, 32, 0, stream>>>(s->rrow_ptr.as<uint32_t>(), s->rcol.as<uint32_t>(),
                                             s->flat_cls[proto.perm].as<FlatLookupClass>(), s->flat_n[proto.perm], proto.stype,
                                             proto.subj, rb_cand_.as<uint32_t>() + 2, cap, d_count);
    ++launches;
    unsigned long long cnt = 0;
    ZG_CUDA(cudaMemcpyAsync(&cnt, d_count, 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if ((flat = cnt <= cap)) {  // more rows than the buffer: the general path
      ++lookups_flat;
      cand = rb_cand_.as<uint32_t>() + 2;
      n = cnt;
    }
  }
  if (!flat) {
    if (s->resources_stale) {
      std::string rerr = gpu_resource_lists(s.get(), stream);
      if (!rerr.empty()) {
        if (err) *err = rerr;
        return ZG_ECUDA;
      }
    }
    n = s->n_resources[res_type];
    cand = s->resources[res_type].as<uint32_t>();
    bool walked = false;
    if (n == 0) {
      // no resource of the type: only the self candidate, if any
    } else if (use_rbfs && proto.stype < s->n_objects.size()) {
      uint64_t nc = 0;
      bool overflow = false;
      if (int rc = lookup_candidates(*s, res_type, proto, &nc, &overflow, err)) return rc;
      if ((walked = !overflow)) {
        ++lookups_rbfs;
        n = nc;
        cand = rb_cand_.as<uint32_t>();
      } else {
        ++lookups_exhaustive;
      }
    } else {
      ++lookups_exhaustive;
    }
    // the exhaustive list is ascending without repeats: the candidates after the cursor are a suffix of it
    sorted = !walked && self == ZG_NO_OBJECT;
  }
  // ---- select: the candidates after the cursor, ascending
  const uint32_t* sel = cand;
  uint64_t m = n;
  uint32_t quiet = ZG_NO_OBJECT;
  const unsigned blk = 256;
  if (sorted) {
    if (has_after && n) {
      lookup_bound_kernel<<<1, 1, 0, stream>>>(cand, n, after, ctrl + 2);
      ++launches;
      ZG_CUDA(cudaMemcpyAsync(h, ctrl, sizeof h, cudaMemcpyDeviceToHost, stream));
      ZG_CUDA(cudaStreamSynchronize(stream));
      sel = cand + h[2];
      m = n - h[2];
    }
  } else {
    const uint64_t n_sel = n + (self != ZG_NO_OBJECT ? 1 : 0);
    if (!lp_sel_.ensure(n_sel * 4 + 4) || !lp_sorted_.ensure(n_sel * 4 + 4)) {
      if (err) *err = "out of device memory (lookup page candidates)";
      return ZG_ENOMEM;
    }
    if (n_sel) {
      lookup_select_kernel<<<static_cast<unsigned>((n_sel + blk - 1) / blk), blk, 0, stream>>>(
          cand, n, has_after ? 1u : 0u, after, self, lp_sel_.as<uint32_t>(), ctrl);
      ++launches;
    }
    ZG_CUDA(cudaMemcpyAsync(h, ctrl, sizeof h, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    m = h[0];
    if (self != ZG_NO_OBJECT && !h[1]) quiet = self;
    sel = lp_sel_.as<uint32_t>();
    if (m > 1) {
      std::string serr = sort_u32(lp_sel_.as<uint32_t>(), lp_sorted_.as<uint32_t>(), m, stream);
      if (!serr.empty()) {
        if (err) *err = serr;
        return ZG_ECUDA;
      }
      sel = lp_sorted_.as<uint32_t>();
    }
  }
  st->after = m;
  if (m == 0) return ZG_OK;
  if (!lp_out_.ensure(std::min(want, m) * 4)) {
    if (err) *err = "out of device memory (lookup page answers)";
    return ZG_ENOMEM;
  }
  ZG_CUDA(cudaMemsetAsync(ctrl, 0, 2 * 8, stream));
  // ---- verify in windows from the front, in id order, until `want` answers are found
  uint64_t found = 0;
  if (flat) {  // every row entry is an answer: one scan takes the first `want` distinct ids
    lookup_window_kernel<<<1, kWindowThreads, 0, stream>>>(sel, m, 0, nullptr, ZG_NO_OBJECT, want, lp_out_.as<uint32_t>(), ctrl);
    ++launches;
    ZG_CUDA(cudaMemcpyAsync(h, ctrl, 2 * 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    found = h[0];
  } else {
    uint64_t pos = 0, w = std::max<uint64_t>(lp_first_, 2 * want);
    for (;;) {
      w = std::min(w, m - pos);
      if (!lk_jobs_.ensure(w * sizeof(zg_check)) || !lk_codes_.ensure(w)) {
        if (err) *err = "out of device memory (lookup page window)";
        return ZG_ENOMEM;
      }
      lookup_fill_kernel<<<static_cast<unsigned>((w + blk - 1) / blk), blk, 0, stream>>>(sel + pos, w, proto, lk_jobs_.as<zg_check>());
      ++launches;
      if (int rc = check_device(lk_jobs_.as<zg_check>(), w, lk_codes_.as<uint8_t>(), stream, true, nullptr, err)) return rc;
      lookup_window_kernel<<<1, kWindowThreads, 0, stream>>>(sel + pos, w, pos > 0 ? 1u : 0u, lk_codes_.as<uint8_t>(), quiet,
                                                             want, lp_out_.as<uint32_t>(), ctrl);
      ++launches;
      uint32_t cflags = 0;
      ZG_CUDA(cudaMemcpyAsync(h, ctrl, 2 * 8, cudaMemcpyDeviceToHost, stream));
      ZG_CUDA(cudaMemcpyAsync(&cflags, ctrl_.as<unsigned long long>() + 3, 4, cudaMemcpyDeviceToHost, stream));
      ZG_CUDA(cudaStreamSynchronize(stream));
      ++st->windows;
      st->verified += w;
      if (cflags & 1u) {
        if (err) *err = "expansion stack overflow (per-warp spill area exhausted)";
        return ZG_ENOMEM;
      }
      if (h[1]) {  // as the unpaged call, but only for a candidate the page's answer depends on
        if (err) *err = "LookupResources: a candidate could not be decided (max dispatch depth / work budget exceeded)";
        return ZG_EDEPTH;
      }
      pos += w;
      found = h[0];
      if (found >= want || pos == m) break;
      // the next window: `growth` times this one at least, and enough for the answers still missing at the density of
      // answers seen so far (with a quarter to spare)
      const uint64_t left = m - pos;
      uint64_t next = std::min(left, w * lp_growth_);
      if (found) {
        const double est = static_cast<double>(want - found) * static_cast<double>(pos) / static_cast<double>(found) * 1.25;
        next = est >= static_cast<double>(left) ? left : std::max(next, static_cast<uint64_t>(est) + 1);
      }
      w = next;
    }
  }
  ids->resize(found);
  if (found) {
    ZG_CUDA(cudaMemcpyAsync(ids->data(), lp_out_.p, found * 4, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
  }
  return ZG_OK;
}


int Device::lookup_batch(const std::vector<LookupReq>& reqs, std::vector<std::vector<uint32_t>>* ids, std::vector<int>* rcs,
                         std::string* err) {
  const size_t K = reqs.size();
  ids->assign(K, {});
  rcs->assign(K, ZG_OK);
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  auto one_by_one = [&]() -> int {
    for (size_t i = 0; i < K; ++i) {
      std::string e1;
      (*rcs)[i] = lookup(reqs[i].res_type, reqs[i].proto, &(*ids)[i], &e1);
      if ((*rcs)[i] && (*rcs)[i] != ZG_EDEPTH) {
        if (err) *err = e1;
        return (*rcs)[i];
      }
    }
    return ZG_OK;
  };
  // the batch buffers overflowed: halves hold about half as much (down to the single path, which degrades to
  // the exhaustive scan by itself)
  auto halves = [&]() -> int {
    const size_t h = K / 2;
    std::vector<LookupReq> a(reqs.begin(), reqs.begin() + h), b(reqs.begin() + h, reqs.end());
    std::vector<std::vector<uint32_t>> ia, ib;
    std::vector<int> ra, rb;
    int rc = lookup_batch(a, &ia, &ra, err);
    if (rc) return rc;
    rc = lookup_batch(b, &ib, &rb, err);
    if (rc) return rc;
    for (size_t i = 0; i < h; ++i) (*ids)[i] = std::move(ia[i]), (*rcs)[i] = ra[i];
    for (size_t i = h; i < K; ++i) (*ids)[i] = std::move(ib[i - h]), (*rcs)[i] = rb[i - h];
    return ZG_OK;
  };
  if (K == 1 || !use_rbfs) return one_by_one();
  if (K > kMaxLookupBatch) return halves();
  const uint64_t cap = lb_cap_;
  for (const auto& r : reqs)
    if (r.res_type >= s->resources.size() || r.proto.stype >= s->n_objects.size()) return one_by_one();
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  const unsigned long long words = (s->total_bits + 31) / 32 + 4;
  constexpr int kLevelsPerRound = 10;
  const size_t n_ctrl = 8 + ZG_MAX_DEPTH + 4 + kMaxLookupBatch;  // flags, cand count, key count, err mask | level counts | per lookup
  if (!rb_visited_.ensure(words * 4 * K) || !rb_front_[0].ensure(cap * 8) || !rb_front_[1].ensure(cap * 8) ||
      !lk_jobs_.ensure(cap * sizeof(zg_check)) || !lb_owner_.ensure(cap) || !lk_codes_.ensure(cap) ||
      !lb_params_.ensure(K * sizeof(LookupParam)) || !lb_ctrl_.ensure(n_ctrl * 8) || !lb_keys_[0].ensure(cap * 8) ||
      !lb_keys_[1].ensure(cap * 8) || !lk_ids_.ensure(cap * 4))
    return one_by_one();  // not enough memory for the batch buffers: the single path scales down by itself
  std::vector<LookupParam> lp(K);
  std::vector<unsigned long long> seeds(K);
  for (size_t i = 0; i < K; ++i) {
    const zg_check& q = reqs[i].proto;
    lp[i] = LookupParam{q.subj, reqs[i].res_type, q.perm, q.stype, q.srel};
    seeds[i] = (static_cast<unsigned long long>(i) << 48) | (static_cast<unsigned long long>(q.stype) << 32) | q.subj;
  }
  unsigned long long* ctrl = lb_ctrl_.as<unsigned long long>();
  unsigned long long* counts = ctrl + 8;
  unsigned long long* per_lookup = counts + ZG_MAX_DEPTH + 4;
  ZG_CUDA(cudaMemsetAsync(ctrl, 0, n_ctrl * 8, stream));
  ZG_CUDA(cudaMemsetAsync(rb_visited_.p, 0, words * 4 * K, stream));
  ZG_CUDA(cudaMemcpyAsync(lb_params_.p, lp.data(), K * sizeof(LookupParam), cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemcpyAsync(rb_front_[0].p, seeds.data(), K * 8, cudaMemcpyHostToDevice, stream));
  const unsigned long long kk = K;
  ZG_CUDA(cudaMemcpyAsync(counts, &kk, 8, cudaMemcpyHostToDevice, stream));
  MrbfsParams p{};
  p.rrow_ptr = s->rrow_ptr.as<uint32_t>();
  p.rcol = s->rcol.as<uint32_t>();
  p.prog = s->prog.as<uint8_t>();
  p.lk = lb_params_.as<LookupParam>();
  p.counts = counts;
  p.cap = cap;
  p.visited = rb_visited_.as<uint32_t>();
  p.words = words;
  p.type_bit_base = s->type_bit_base.as<unsigned long long>();
  p.cand = lk_jobs_.as<zg_check>();
  p.cand_owner = lb_owner_.as<uint8_t>();
  p.cand_count = ctrl + 1;
  p.cand_cap = cap;
  p.flags = reinterpret_cast<uint32_t*>(ctrl);
  unsigned long long host[4] = {0, 0, 0, 0};
  int level = 0, cur = 0;
  for (;;) {
    // a round of levels without a host round trip: a level whose input is empty costs one empty launch
    for (int r = 0; r < kLevelsPerRound && level <= ZG_MAX_DEPTH + 1; ++r, ++level) {
      p.in = rb_front_[cur].as<unsigned long long>();
      p.out = rb_front_[cur ^ 1].as<unsigned long long>();
      p.level = level;
      mrbfs_expand_kernel<<<sm_count_ * 8, 256, 0, stream>>>(p);
      ++launches;
      cur ^= 1;
    }
    unsigned long long last = 0;
    ZG_CUDA(cudaMemcpyAsync(host, ctrl, sizeof host, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaMemcpyAsync(&last, counts + level, 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if (static_cast<uint32_t>(host[0]) & 16u) return halves();  // frontier / candidate buffers overflowed
    if (last == 0 || level > ZG_MAX_DEPTH + 1) break;  // deeper objects cannot be within the dispatch cap anyway
  }
  const uint64_t n_cand = host[1];
  lookup_batches += 1;
  lookups_batched += K;
  if (n_cand == 0) return ZG_OK;
  int rc = check_device(lk_jobs_.as<zg_check>(), n_cand, lk_codes_.as<uint8_t>(), stream, true, nullptr, err);
  if (rc) return rc;
  const unsigned blk = 256, grid = static_cast<unsigned>((n_cand + blk - 1) / blk);
  lookup_keys_kernel<<<grid, blk, 0, stream>>>(lk_jobs_.as<zg_check>(), lb_owner_.as<uint8_t>(), lk_codes_.as<uint8_t>(), n_cand,
                                               lb_keys_[0].as<unsigned long long>(), ctrl + 2, per_lookup, ctrl + 3);
  ++launches;
  std::vector<unsigned long long> cnt(K);
  uint32_t cflags = 0;
  ZG_CUDA(cudaMemcpyAsync(host, ctrl, sizeof host, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(cnt.data(), per_lookup, K * 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(&cflags, ctrl_.as<unsigned long long>() + 3, 4, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  if (cflags & 1u) {
    if (err) *err = "expansion stack overflow (per-warp spill area exhausted)";
    return ZG_ENOMEM;
  }
  const uint64_t n_keys = host[2];
  const unsigned long long err_mask = host[3];
  if (n_keys) {
    // ascending (lookup, id): one radix sort over the 32 id bits and the few lookup bits
    int kbits = 1;
    while ((1u << kbits) < K) ++kbits;
    std::string serr = sort_u64(lb_keys_[0].as<unsigned long long>(), lb_keys_[1].as<unsigned long long>(), n_keys, 32 + kbits, stream);
    if (!serr.empty()) {
      if (err) *err = serr;
      return ZG_ECUDA;
    }
    low_words_kernel<<<static_cast<unsigned>((n_keys + blk - 1) / blk), blk, 0, stream>>>(lb_keys_[1].as<unsigned long long>(),
                                                                                      n_keys, lk_ids_.as<uint32_t>());
    ++launches;
    // one copy back into pinned memory, then split per lookup
    if (pin_lk_cap_ < n_keys * 4) {
      if (pin_lk_) cudaFreeHost(pin_lk_);
      pin_lk_cap_ = 0;
      ZG_CUDA(cudaMallocHost(&pin_lk_, n_keys * 4 + (n_keys * 4) / 4));
      pin_lk_cap_ = n_keys * 4 + (n_keys * 4) / 4;
    }
    ZG_CUDA(cudaMemcpyAsync(pin_lk_, lk_ids_.p, n_keys * 4, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    uint64_t off = 0;
    for (size_t i = 0; i < K; ++i) {
      const uint32_t* src = static_cast<const uint32_t*>(pin_lk_) + off;
      (*ids)[i].assign(src, src + cnt[i]);
      off += cnt[i];
    }
  }
  for (size_t i = 0; i < K; ++i)
    if ((err_mask >> i) & 1ull) {
      (*rcs)[i] = ZG_EDEPTH;
      (*ids)[i].clear();
    }
  return ZG_OK;
}

int Device::lookup_subjects(uint16_t res_type, uint32_t res, uint16_t perm, uint16_t stype, uint16_t srel,
                            bool include_wildcard, SubjectsAnswer* ans, std::string* err) {
  *ans = SubjectsAnswer{};
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  if (res_type >= s->n_objects.size() || stype >= s->n_objects.size()) {
    if (err) *err = "unknown resource or subject type";
    return ZG_EINVAL;
  }
  if (res >= s->n_objects[res_type]) return ZG_OK;  // never written: no relationship names it
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  zg_check proto{};
  proto.res = res;
  proto.perm = perm;
  proto.stype = stype;
  proto.srel = srel;
  const size_t n_ctrl = 8 + ZG_MAX_DEPTH + 4;  // [0] flags, [1] candidates, [2] HAS, [3] NO, [4] concrete, [5] scratch | level counts
  if (!ls_ctrl_.ensure(n_ctrl * 8)) {
    if (err) *err = "out of device memory (lookup)";
    return ZG_ENOMEM;
  }
  unsigned long long* ctrl = ls_ctrl_.as<unsigned long long>();
  unsigned long long* counts = ctrl + 8;
  uint32_t* lflags = reinterpret_cast<uint32_t*>(ctrl);
  ZG_CUDA(cudaMemsetAsync(ctrl, 0, n_ctrl * 8, stream));
  uint64_t n = 0;  // items of the first verification, the probe included
  bool walked = false;
  const uint64_t cap = rb_cap_;
  const unsigned long long words = (s->total_bits + 31) / 32 + 4;
  if (use_rbfs && rb_visited_.ensure(words * 4) && rb_front_[0].ensure(cap * 8) && rb_front_[1].ensure(cap * 8) &&
      ls_jobs_.ensure((cap + 2) * sizeof(zg_check))) {
    ZG_CUDA(cudaMemsetAsync(rb_visited_.p, 0, words * 4, stream));
    FwalkParams p{};
    p.row_ptr = s->row_ptr.as<uint32_t>();
    p.col = s->col.as<uint32_t>();
    p.fwd = s->ls_fwd.as<FwdClass>();
    p.type_off = s->ls_type_off.as<uint32_t>();
    p.mask = s->ls_mask.as<uint32_t>() + static_cast<size_t>(perm) * s->ls_mask_words;
    p.counts = counts;
    p.cap = cap;
    p.visited = rb_visited_.as<uint32_t>();
    p.type_bit_base = s->type_bit_base.as<unsigned long long>();
    p.proto = proto;
    p.cand = ls_jobs_.as<zg_check>();
    p.cand_count = ctrl + 1;
    p.cand_cap = cap + 2;
    p.flags = lflags;
    p.in = rb_front_[0].as<unsigned long long>();
    fwalk_seed_kernel<<<1, 32, 0, stream>>>(p, res_type);
    ++launches;
    constexpr int kLevelsPerRound = 10;
    int level = 0, cur = 0;
    for (;;) {
      // a round of levels without a host round trip: a level whose input is empty costs one empty launch
      for (int r = 0; r < kLevelsPerRound && level <= ZG_MAX_DEPTH + 1; ++r, ++level) {
        p.in = rb_front_[cur].as<unsigned long long>();
        p.out = rb_front_[cur ^ 1].as<unsigned long long>();
        p.level = level;
        fwalk_expand_kernel<<<sm_count_ * 8, 256, 0, stream>>>(p);
        ++launches;
        cur ^= 1;
      }
      unsigned long long host[2] = {0, 0}, last = 0;
      ZG_CUDA(cudaMemcpyAsync(host, ctrl, sizeof host, cudaMemcpyDeviceToHost, stream));
      ZG_CUDA(cudaMemcpyAsync(&last, counts + level, 8, cudaMemcpyDeviceToHost, stream));
      ZG_CUDA(cudaStreamSynchronize(stream));
      if (static_cast<uint32_t>(host[0]) & 16u) break;  // frontier / candidate buffers overflowed: verify every object
      if (last == 0 || level > ZG_MAX_DEPTH + 1) {      // deeper objects cannot be within the dispatch cap anyway
        walked = true;
        n = host[1];
        break;
      }
    }
  }
  if (walked) {
    ++subject_lookups_walk;
  } else {
    const uint64_t no = s->n_objects[stype];
    n = no + 1;
    if (!ls_jobs_.ensure(n * sizeof(zg_check))) {
      if (err) *err = "out of device memory (lookup)";
      return ZG_ENOMEM;
    }
    ls_fill_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(proto, no, ls_jobs_.as<zg_check>());
    ++launches;
    ++subject_lookups_exhaustive;
  }
  ans->fell_back = !walked;
  ans->n_verified = n;
  subject_items_verified += n;
  if (!ls_codes_.ensure(n) || !ls_has_.ensure(n * sizeof(zg_check)) || !ls_ids_.ensure(n * 16 + 64)) {
    if (err) *err = "out of device memory (lookup)";
    return ZG_ENOMEM;
  }
  uint32_t* has_ids = ls_ids_.as<uint32_t>();
  uint32_t* no_ids = has_ids + n;
  uint32_t* out_ids = no_ids + n;
  uint32_t* tmp_ids = out_ids + n;
  uint8_t* codes = ls_codes_.as<uint8_t>();
  int rc = check_device(ls_jobs_.as<zg_check>(), n, codes, stream, true, nullptr, err);
  if (rc) return rc;
  if (n > 1) {
    ls_split_kernel<<<static_cast<unsigned>((n - 1 + 255) / 256), 256, 0, stream>>>(
        ls_jobs_.as<zg_check>(), codes, n, has_ids, ls_has_.as<zg_check>(), no_ids, ctrl + 2, lflags);
    ++launches;
  }
  uint8_t probe = 0;
  unsigned long long hc[4] = {0, 0, 0, 0};
  uint32_t cflags = 0;
  ZG_CUDA(cudaMemcpyAsync(&probe, codes, 1, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(hc, ctrl, sizeof hc, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(&cflags, ctrl_.as<unsigned long long>() + 3, 4, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  if (cflags & 1u) {
    if (err) *err = "expansion stack overflow (per-warp spill area exhausted)";
    return ZG_ENOMEM;
  }
  if (probe == ZG_ITEM_ERROR || (static_cast<uint32_t>(hc[0]) & 8u)) {
    // as LookupResources: a silently shortened answer would read as "not allowed"
    if (err) *err = "LookupSubjects: a subject could not be decided (max dispatch depth / work budget exceeded)";
    return ZG_EDEPTH;
  }
  const uint64_t n_has = hc[2], n_no = hc[3];
  const bool granted = srel == kNone && probe == ZG_HAS_PERMISSION;
  const uint32_t* concrete = has_ids;
  uint64_t n_concrete = n_has;
  if (granted && n_has) {
    // The wildcard is granted: list the subjects that also check HAS with every wildcard relationship
    // invisible. An undecidable one is only "not listed": it checked HAS, the wildcard covers it.
    no_wildcards_ = true;
    rc = check_device(ls_has_.as<zg_check>(), n_has, codes, stream, true, nullptr, err);
    no_wildcards_ = false;
    if (rc) return rc;
    lookup_compact_kernel<<<static_cast<unsigned>((n_has + 255) / 256), 256, 0, stream>>>(
        has_ids, codes, n_has, out_ids, n_has, ctrl + 4, reinterpret_cast<uint32_t*>(ctrl + 5));
    ++launches;
    unsigned long long cnt = 0;
    ZG_CUDA(cudaMemcpyAsync(&cnt, ctrl + 4, 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaMemcpyAsync(&cflags, ctrl_.as<unsigned long long>() + 3, 4, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if (cflags & 1u) {
      if (err) *err = "expansion stack overflow (per-warp spill area exhausted)";
      return ZG_ENOMEM;
    }
    concrete = out_ids;
    n_concrete = cnt;
  }
  ans->wildcard = granted && include_wildcard;
  // ascending ids: radix sort on the device when the list is large
  auto fetch = [&](const uint32_t* d, uint64_t cnt, std::vector<uint32_t>* out) -> int {
    out->resize(cnt);
    if (!cnt) return ZG_OK;
    const uint32_t* src = d;
    if (cnt > 2048) {
      std::string serr = sort_u32(d, tmp_ids, cnt, stream);
      if (!serr.empty()) {
        if (err) *err = serr;
        return ZG_ECUDA;
      }
      src = tmp_ids;
    }
    ZG_CUDA(cudaMemcpyAsync(out->data(), src, cnt * 4, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    if (cnt <= 2048) std::sort(out->begin(), out->end());
    return ZG_OK;
  };
  rc = fetch(concrete, n_concrete, &ans->ids);
  if (!rc && ans->wildcard) rc = fetch(no_ids, n_no, &ans->excluded);
  return rc;
}

// ---- relationship filters (filter.cuh) --------------------------------------------------------

static unsigned ingress_grid(uint64_t n, int sm_count);  // device ingress, below

// The classes whose relation, subject type and subject relation agree with the filter, in data-relation order.
static void select_classes(const Schema& sc, const Snapshot& s, const Store::Filter& f, std::vector<FilterSel>* sel) {
  sel->clear();
  for (size_t ri = 0; ri < sc.rel_slots.size() && ri < s.rels.size(); ++ri) {
    const int slot = sc.rel_slots[ri];
    if ((f.res_type >= 0 && sc.slots[slot].type != f.res_type) || (f.rel >= 0 && slot != f.rel)) continue;
    const DRel& r = s.rels[ri];
    for (uint16_t k = 0; k < r.ncls; ++k) {
      const DCls& c = s.cls[r.cls_begin + k];
      if (f.subj_type >= 0 && c.stype != f.subj_type) continue;
      if (f.subj_wildcard && c.sslot != kWildcard) continue;
      if (f.has_subj && c.sslot == kWildcard) continue;  // a concrete id never matches a wildcard relationship
      if (f.has_srel && c.sslot != f.srel) continue;
      FilterSel x{};
      x.row_base = r.row_base + k;
      x.rrow_base = c.rrow_base;
      x.nres = r.nres;
      x.nsubj = c.nsubj;
      x.stride = r.stride;
      x.rstride = c.rstride;
      x.rel = static_cast<uint16_t>(slot);
      x.stype = c.stype;
      x.srel = c.sslot;
      x.pos = static_cast<uint16_t>(page_class_pos(sc, slot, c.stype, c.sslot));
      x.rtype = sc.slots[slot].type;
      sel->push_back(x);
    }
  }
}

// The bitmap of every selected class: its resource type's (px->type).
static std::vector<const uint32_t*> class_bits(const PrefixBits& px, const std::vector<FilterSel>& sel) {
  std::vector<const uint32_t*> bits(sel.size());
  for (size_t k = 0; k < sel.size(); ++k) bits[k] = px.type[sel[k].rtype];
  return bits;
}

int Device::match_filter(const Schema& sc, const Store::Filter& f, uint32_t now, uint64_t* count, std::vector<zg_tuple>* tuples,
                         std::vector<uint32_t>* expires, bool* too_big, std::string* err, const PrefixBits* px) {
  *count = 0;
  *too_big = false;
  if (tuples) tuples->clear();
  if (expires) expires->clear();
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  if (f.impossible) return ZG_OK;
  std::vector<FilterSel> sel;
  select_classes(sc, *s, f, &sel);
  if (sel.empty() || s->n_tuples == 0) return ZG_OK;
  FilterPlan p{};
  p.has_subj = f.has_subj;
  p.res = f.res;
  p.subj = f.has_subj ? f.subj : 0;
  p.now = now;
  if (!px) return run_filter(sc, *s, sel, p, filter_shape(f), false, count, tuples, expires, too_big, err);
  const std::vector<const uint32_t*> bits = class_bits(*px, sel);
  return run_filter(sc, *s, sel, p, filter_shape(f), false, count, tuples, expires, too_big, err, &bits, px->bytes);
}

int Device::match_expired(const Schema& sc, uint32_t before, uint64_t* count, std::vector<zg_tuple>* tuples, bool* too_big,
                          std::string* err) {
  *count = 0;
  *too_big = false;
  if (tuples) tuples->clear();
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  // every class whose relationships may carry an expiration; the rows of any other class hold none
  std::vector<FilterSel> sel;
  for (size_t ri = 0; ri < sc.rel_slots.size() && ri < s->rels.size(); ++ri) {
    const DRel& r = s->rels[ri];
    for (uint16_t k = 0; k < r.ncls; ++k) {
      const DCls& c = s->cls[r.cls_begin + k];
      if (!(c.flags & CF_EXPIRY)) continue;
      FilterSel x{};
      x.row_base = r.row_base + k;
      x.nres = r.nres;
      x.stride = r.stride;
      x.rel = static_cast<uint16_t>(sc.rel_slots[ri]);
      x.stype = c.stype;
      x.srel = c.sslot;
      sel.push_back(x);
    }
  }
  if (sel.empty() || s->n_tuples == 0) return ZG_OK;
  FilterPlan p{};
  p.now = before;
  return run_filter(sc, *s, sel, p, kByScan, true, count, tuples, nullptr, too_big, err);
}

int Device::run_filter(const Schema& sc, const Snapshot& s, const std::vector<FilterSel>& sel, FilterPlan& p, FilterShape shape,
                       bool expired, uint64_t* count, std::vector<zg_tuple>* tuples, std::vector<uint32_t>* expires,
                       bool* too_big, std::string* err, const std::vector<const uint32_t*>* bits, uint64_t held) {
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  if (!flt_ctrl_.ensure(8)) {
    if (err) *err = "out of device memory (filter)";
    return ZG_ENOMEM;
  }
  p.row_ptr = s.row_ptr.as<uint32_t>();
  p.col = s.col.as<uint32_t>();
  p.exp = sc.has_expiry ? s.exp.as<uint32_t>() : nullptr;
  p.rrow_ptr = s.rrow_ptr.as<uint32_t>();
  p.rcol = s.rcol.as<uint32_t>();
  p.count = flt_ctrl_.as<unsigned long long>();
  // every selected class, kMaxFilterSel per launch; the launches append behind one count
  auto run = [&](bool emit) -> int {
    ZG_CUDA(cudaMemsetAsync(p.count, 0, 8, stream));
    const unsigned grid = static_cast<unsigned>(sm_count_) * 8;
    for (size_t at = 0; at < sel.size(); at += kMaxFilterSel) {
      p.n_sel = static_cast<uint32_t>(std::min<size_t>(kMaxFilterSel, sel.size() - at));
      std::copy(sel.begin() + at, sel.begin() + at + p.n_sel, p.sel);
      if (bits) {  // a prefix: the resource shape never has one (res_id and a prefix are refused together)
        std::copy(bits->begin() + at, bits->begin() + at + p.n_sel, p.bits);
        if (shape == kBySubject) {
          if (emit) filter_subject_kernel<true, true><<<grid, kFilterThreads, 0, stream>>>(p);
          else filter_subject_kernel<false, true><<<grid, kFilterThreads, 0, stream>>>(p);
        } else {
          if (emit) filter_scan_kernel<true, true><<<grid, kFilterThreads, 0, stream>>>(p);
          else filter_scan_kernel<false, true><<<grid, kFilterThreads, 0, stream>>>(p);
        }
      } else if (expired) {
        if (emit) filter_expired_kernel<true><<<grid, kFilterThreads, 0, stream>>>(p);
        else filter_expired_kernel<false><<<grid, kFilterThreads, 0, stream>>>(p);
      } else if (shape == kByResource) {
        if (emit) filter_resource_kernel<true><<<grid, kFilterThreads, 0, stream>>>(p);
        else filter_resource_kernel<false><<<grid, kFilterThreads, 0, stream>>>(p);
      } else if (shape == kBySubject) {
        if (emit) filter_subject_kernel<true><<<grid, kFilterThreads, 0, stream>>>(p);
        else filter_subject_kernel<false><<<grid, kFilterThreads, 0, stream>>>(p);
      } else {
        if (emit) filter_scan_kernel<true><<<grid, kFilterThreads, 0, stream>>>(p);
        else filter_scan_kernel<false><<<grid, kFilterThreads, 0, stream>>>(p);
      }
      ++launches;
    }
    ZG_CUDA(cudaGetLastError());
    return ZG_OK;
  };
  if (int rc = run(false)) return rc;
  unsigned long long n = 0;
  ZG_CUDA(cudaMemcpyAsync(&n, p.count, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  *count = n;
  if (!tuples || n == 0) return ZG_OK;
  size_t free_b = 0, total_b = 0;
  ZG_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const size_t bytes = n * (sizeof(zg_tuple) + 4);
  if (bytes > flt_out_.cap + flt_exp_.cap && bytes + held > free_b / 4) {
    *too_big = true;
    return ZG_OK;
  }
  if (!flt_out_.ensure(n * sizeof(zg_tuple)) || !flt_exp_.ensure(n * 4)) {
    if (err) *err = "out of device memory (filter output)";
    return ZG_ENOMEM;
  }
  p.out = flt_out_.as<zg_tuple>();
  p.out_exp = flt_exp_.as<uint32_t>();
  p.cap = n;
  if (int rc = run(true)) return rc;
  unsigned long long n2 = 0;
  tuples->resize(n);
  if (expires) expires->resize(n);
  ZG_CUDA(cudaMemcpyAsync(&n2, p.count, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(tuples->data(), p.out, n * sizeof(zg_tuple), cudaMemcpyDeviceToHost, stream));
  if (expires) ZG_CUDA(cudaMemcpyAsync(expires->data(), p.out_exp, n * 4, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  if (n2 != n) {  // the snapshot cannot change under the device lock
    if (err) *err = "filter: the emit launch found " + std::to_string(n2) + " relationships, the count launch " + std::to_string(n);
    return ZG_ECUDA;
  }
  return ZG_OK;
}

int Device::page_filter(const Schema& sc, const Store::Filter& f, uint32_t now, const PageKey* after, uint64_t want,
                        std::vector<zg_tuple>* tuples, std::vector<uint32_t>* expires, PageStats* st, bool* too_big,
                        std::string* err, const PrefixBits* px) {
  tuples->clear();
  expires->clear();
  *too_big = false;
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  if (f.impossible || want == 0) return ZG_OK;
  std::vector<FilterSel> sel;
  select_classes(sc, *s, f, &sel);
  if (sel.empty() || s->n_tuples == 0) return ZG_OK;
  std::sort(sel.begin(), sel.end(), [](const FilterSel& a, const FilterSel& b) {
    return a.rtype != b.rtype ? a.rtype < b.rtype : a.pos < b.pos;
  });
  const FilterShape shape = filter_shape(f);
  // the output: `want` records (the subject shape: a segment of them per selected class), within a quarter of the free
  // memory; one type's classes go into one plan
  size_t free_b = 0, total_b = 0;
  ZG_CUDA(cudaSetDevice(device));
  ZG_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const uint64_t segs = shape == kBySubject ? sel.size() : 1;
  const uint64_t bytes = segs * want * (sizeof(zg_tuple) + 4);
  // a prefix: its bitmaps, and for the scan shape the largest match list (ids, entries, their sums, the word scan)
  uint64_t held = 0;
  if (px) {
    held = px->bytes;
    if (shape == kByScan)
      for (const FilterSel& x : sel) held = std::max<uint64_t>(held, px->bytes + uint64_t(px->n_ids[x.rtype]) * 24 + (1u << 20));
  }
  bool fits = bytes <= flt_out_.cap + flt_exp_.cap ? held <= free_b / 4 : bytes + held <= free_b / 4;
  for (size_t g = 0, g0 = 0; fits && g <= sel.size(); ++g)
    if (g == sel.size() || sel[g].rtype != sel[g0].rtype) {
      fits = shape == kBySubject || g - g0 <= static_cast<size_t>(kMaxFilterSel);
      g0 = g;
    }
  if (!fits) {
    *too_big = true;
    return ZG_OK;
  }
  if (!flt_out_.ensure(segs * want * sizeof(zg_tuple)) || !flt_exp_.ensure(segs * want * 4) || !flt_ctrl_.ensure(64)) {
    if (err) *err = "out of device memory (page output)";
    return ZG_ENOMEM;
  }
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  PagePlan p{};
  p.row_ptr = s->row_ptr.as<uint32_t>();
  p.col = s->col.as<uint32_t>();
  p.exp = sc.has_expiry ? s->exp.as<uint32_t>() : nullptr;
  p.rrow_ptr = s->rrow_ptr.as<uint32_t>();
  p.rcol = s->rcol.as<uint32_t>();
  p.now = now;
  p.has_subj = f.has_subj;
  p.subj = f.has_subj ? f.subj : 0;
  zg_tuple* d_out = flt_out_.as<zg_tuple>();
  uint32_t* d_exp = flt_exp_.as<uint32_t>();
  unsigned long long* ctrl = flt_ctrl_.as<unsigned long long>();

  if (shape == kBySubject) {  // one warp per class, its segment of `want`; merged on the host (page_merge)
    page_set_after(p, after);
    p.want = want;
    if (!pg_seg_.ensure(sel.size() * 4)) {
      if (err) *err = "out of device memory (page segments)";
      return ZG_ENOMEM;
    }
    for (size_t at = 0; at < sel.size(); at += kMaxFilterSel) {
      p.n_sel = static_cast<uint32_t>(std::min<size_t>(kMaxFilterSel, sel.size() - at));
      std::copy(sel.begin() + at, sel.begin() + at + p.n_sel, p.sel);
      p.out = d_out + at * want;
      p.out_exp = d_exp + at * want;
      p.seg_count = pg_seg_.as<uint32_t>() + at;
      if (px) {
        for (uint32_t k = 0; k < p.n_sel; ++k) p.bits[k] = px->type[p.sel[k].rtype];
        page_subject_kernel<true><<<p.n_sel, 32, 0, stream>>>(p);
      } else {
        page_subject_kernel<<<p.n_sel, 32, 0, stream>>>(p);
      }
      ++st->launches;
    }
    ZG_CUDA(cudaGetLastError());
    std::vector<uint32_t> seg(sel.size());
    ZG_CUDA(cudaMemcpyAsync(seg.data(), pg_seg_.p, seg.size() * 4, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    std::vector<zg_tuple> rec(sel.size() * want);
    std::vector<uint32_t> rec_exp(sel.size() * want);
    for (size_t k = 0; k < sel.size(); ++k) {
      if (!seg[k]) continue;
      ZG_CUDA(cudaMemcpyAsync(rec.data() + k * want, d_out + k * want, seg[k] * sizeof(zg_tuple), cudaMemcpyDeviceToHost, stream));
      ZG_CUDA(cudaMemcpyAsync(rec_exp.data() + k * want, d_exp + k * want, seg[k] * 4ull, cudaMemcpyDeviceToHost, stream));
      st->scanned += seg[k];
    }
    ZG_CUDA(cudaStreamSynchronize(stream));
    page_merge(sel, seg.data(), rec.data(), rec_exp.data(), want, tuples, expires);
    return ZG_OK;
  }

  // scan and resource shapes: windows of one type's objects (page_walk)
  struct Ops {
    Device* d;
    unsigned long long* ctrl;
    zg_tuple* out;
    uint32_t* out_exp;
    PageStats* st;
    std::string* err;
    const PrefixBits* px;
    int list_type = -1;  // a prefix: the type whose match list px_ids_ / px_sum_ hold
    uint32_t list_m = 0;
    // A prefix page: the ascending ids of the type's matches and the exclusive sum of their entries in the block.
    int build_list(const PagePlan& p, unsigned long long block, uint32_t stride) {
      const int type = p.sel[0].rtype;
      const uint32_t n_ids = px->n_ids[type], words = (n_ids + 31) / 32, nres = p.sel[0].nres;
      const uint32_t* bits = px->type[type];
      size_t t1 = 0, t2 = 0;
      cub::DeviceScan::ExclusiveSum(nullptr, t1, d->px_first_.as<uint32_t>(), d->px_first_.as<uint32_t>(),
                                    static_cast<int64_t>(words) + 1, d->stream);
      cub::DeviceScan::ExclusiveSum(nullptr, t2, d->px_ent_.as<unsigned long long>(), d->px_sum_.as<unsigned long long>(),
                                    static_cast<int64_t>(n_ids) + 1, d->stream);
      if (!d->px_first_.ensure((uint64_t(words) + 1) * 4) || !d->px_ids_.ensure((uint64_t(n_ids) + 1) * 4) ||
          !d->px_ent_.ensure((uint64_t(n_ids) + 1) * 8) || !d->px_sum_.ensure((uint64_t(n_ids) + 1) * 8) ||
          !d->px_tmp_.ensure(std::max(t1, t2))) {
        if (err) *err = "out of device memory (prefix match list)";
        return ZG_ENOMEM;
      }
      uint32_t* first = d->px_first_.as<uint32_t>();
      const unsigned grid = ingress_grid(uint64_t(words) + 1, d->sm_count_);
      prefix_word_count_kernel<<<grid, kFilterThreads, 0, d->stream>>>(bits, words, first);
      ZG_CUDA(cudaGetLastError());
      if (cub::DeviceScan::ExclusiveSum(d->px_tmp_.p, t1, first, first, static_cast<int64_t>(words) + 1, d->stream) != cudaSuccess) {
        if (err) *err = "page: the scan of the prefix bitmap failed";
        return ZG_ECUDA;
      }
      uint32_t m = 0;
      ZG_CUDA(cudaMemcpyAsync(&m, first + words, 4, cudaMemcpyDeviceToHost, d->stream));
      prefix_list_kernel<<<grid, kFilterThreads, 0, d->stream>>>(bits, words, first, p.row_ptr, block, stride, nres,
                                                                d->px_ids_.as<uint32_t>(), d->px_ent_.as<unsigned long long>());
      ZG_CUDA(cudaGetLastError());
      ZG_CUDA(cudaStreamSynchronize(d->stream));
      if (cub::DeviceScan::ExclusiveSum(d->px_tmp_.p, t2, d->px_ent_.as<unsigned long long>(), d->px_sum_.as<unsigned long long>(),
                                        static_cast<int64_t>(m) + 1, d->stream) != cudaSuccess) {
        if (err) *err = "page: the scan of the prefix match list failed";
        return ZG_ECUDA;
      }
      st->launches += 4;
      st->list_launches += 4;
      list_type = type;
      list_m = m;
      return ZG_OK;
    }
    int window(const PagePlan& p, unsigned long long block, uint32_t stride, uint32_t obj0, unsigned long long entries,
               uint32_t* obj1, unsigned long long* n) {
      if (px) {
        if (list_type != p.sel[0].rtype)
          if (int rc = build_list(p, block, stride)) return rc;
        prefix_window_kernel<<<1, 32, 0, d->stream>>>(d->px_ids_.as<uint32_t>(), d->px_sum_.as<unsigned long long>(), list_m,
                                                      obj0, p.sel[0].nres, entries, ctrl);
        ++st->list_launches;
      } else {
        page_window_kernel<<<1, 32, 0, d->stream>>>(p.row_ptr, block, stride, obj0, p.sel[0].nres, entries, ctrl);
      }
      ++st->launches;
      ZG_CUDA(cudaGetLastError());
      unsigned long long h[2];
      ZG_CUDA(cudaMemcpyAsync(h, ctrl, 16, cudaMemcpyDeviceToHost, d->stream));
      ZG_CUDA(cudaStreamSynchronize(d->stream));
      *obj1 = static_cast<uint32_t>(h[0]);
      *n = h[1];
      return ZG_OK;
    }
    int tiles(PagePlan& p, unsigned long long got, unsigned long long* total) {
      const uint64_t n_tiles = (uint64_t(p.obj1 - p.obj0) + 31) / 32;
      size_t tmp = 0;
      cub::DeviceScan::ExclusiveSum(nullptr, tmp, d->pg_count_.as<unsigned long long>(), d->pg_off_.as<unsigned long long>(),
                                    static_cast<int64_t>(n_tiles + 1), d->stream);
      if (!d->pg_count_.ensure((n_tiles + 1) * 8) || !d->pg_off_.ensure((n_tiles + 1) * 8) || !d->pg_tmp_.ensure(tmp)) {
        if (err) *err = "out of device memory (page tiles)";
        return ZG_ENOMEM;
      }
      p.tile_count = d->pg_count_.as<unsigned long long>();
      p.tile_off = d->pg_off_.as<unsigned long long>();
      p.out = out + got;
      p.out_exp = out_exp + got;
      const uint64_t warps_per_block = kFilterThreads / 32;
      const unsigned grid = static_cast<unsigned>(
          std::max<uint64_t>(1, std::min<uint64_t>((n_tiles + warps_per_block - 1) / warps_per_block, uint64_t(d->sm_count_) * 16)));
      ZG_CUDA(cudaMemsetAsync(p.tile_count + n_tiles, 0, 8, d->stream));
      if (px) page_count_kernel<true><<<grid, kFilterThreads, 0, d->stream>>>(p);
      else page_count_kernel<<<grid, kFilterThreads, 0, d->stream>>>(p);
      ZG_CUDA(cudaGetLastError());
      if (cub::DeviceScan::ExclusiveSum(d->pg_tmp_.p, tmp, p.tile_count, d->pg_off_.as<unsigned long long>(),
                                        static_cast<int64_t>(n_tiles + 1), d->stream) != cudaSuccess) {
        if (err) *err = "page: the scan of the tile counts failed";
        return ZG_ECUDA;
      }
      if (px) page_emit_kernel<true><<<grid, kFilterThreads, 0, d->stream>>>(p);
      else page_emit_kernel<<<grid, kFilterThreads, 0, d->stream>>>(p);
      ZG_CUDA(cudaGetLastError());
      st->launches += 3;
      ZG_CUDA(cudaMemcpyAsync(total, p.tile_off + n_tiles, 8, cudaMemcpyDeviceToHost, d->stream));
      ZG_CUDA(cudaStreamSynchronize(d->stream));
      return ZG_OK;
    }
  } ops{this, ctrl, d_out, d_exp, st, err, px};
  unsigned long long got = 0;
  std::vector<const uint32_t*> bits;
  if (px) bits = class_bits(*px, sel);
  if (int rc = page_walk(ops, p, sel, shape == kByResource, f.res, after, want, &got, &st->scanned, px ? &bits : nullptr))
    return rc;
  tuples->resize(got);
  expires->resize(got);
  if (got) {
    ZG_CUDA(cudaMemcpyAsync(tuples->data(), d_out, got * sizeof(zg_tuple), cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaMemcpyAsync(expires->data(), d_exp, got * 4, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
  }
  return ZG_OK;
}

int Device::scan_mentions(const Schema& sc, Store::IdBits* bits, std::string* err) {
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  std::vector<MentionType> types;
  const uint64_t words = mention_types(sc, s->rels, s->cls, s->n_objects, &types);
  if (bits->size() < types.size()) bits->resize(types.size());
  if (words == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  if (!mention_bits_.ensure(words * 4)) {
    if (err) *err = "out of device memory (mention bitmaps)";
    return ZG_ENOMEM;
  }
  MentionPlan p{};
  p.row_ptr = s->row_ptr.as<uint32_t>();
  p.rrow_ptr = s->rrow_ptr.as<uint32_t>();
  p.bits = mention_bits_.as<uint32_t>();
  const uint64_t want = (words + kFilterThreads / 32 - 1) / (kFilterThreads / 32);
  const unsigned grid = static_cast<unsigned>(std::max<uint64_t>(1, std::min<uint64_t>(want, uint64_t(sm_count_) * 8)));
  for (size_t at = 0; at < types.size(); at += kMaxMentionTypes) {
    p.n_types = static_cast<uint32_t>(std::min<size_t>(kMaxMentionTypes, types.size() - at));
    std::copy(types.begin() + at, types.begin() + at + p.n_types, p.type);
    mention_scan_kernel<<<grid, kFilterThreads, 0, stream>>>(p);
    ++launches;
  }
  ZG_CUDA(cudaGetLastError());
  std::vector<uint32_t> host(words);
  ZG_CUDA(cudaMemcpyAsync(host.data(), p.bits, words * 4, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  for (size_t t = 0; t < types.size(); ++t) {
    const uint64_t n = (uint64_t(types[t].n_ids) + 31) / 32;
    std::vector<uint32_t>& b = (*bits)[t];
    if (b.size() < n) b.resize(n, 0);
    for (uint64_t i = 0; i < n; ++i) b[i] |= host[types[t].word0 + i];
  }
  return ZG_OK;
}

// ---- resource id prefixes ---------------------------------------------------------------------

int Device::prefix_scan(const Store& store, const Schema& sc, int res_type, const std::string& prefix, PrefixBits* out,
                        PrefixStats* st, bool* too_big, std::string* err) {
  *too_big = false;
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  // the types a filter of res_type may select, each covering the larger of its object capacity and its rows
  const size_t nt = sc.types.size();
  out->type.assign(nt, nullptr);
  out->n_ids.assign(nt, 0);
  std::vector<uint64_t> word0(nt, 0);
  std::vector<char> want(nt, 0);
  for (size_t ri = 0; ri < sc.rel_slots.size() && ri < s->rels.size(); ++ri) {
    const int t = sc.slots[sc.rel_slots[ri]].type;
    if (res_type >= 0 && t != res_type) continue;
    want[t] = 1;
    out->n_ids[t] = std::max(out->n_ids[t], s->rels[ri].nres);
  }
  uint64_t words = 0;
  for (size_t t = 0; t < nt; ++t) {
    if (!want[t]) continue;
    if (t < s->n_objects.size()) out->n_ids[t] = std::max(out->n_ids[t], s->n_objects[t]);
    word0[t] = words;
    words += (uint64_t(out->n_ids[t]) + 31) / 32;
  }
  out->bytes = words * 4;
  ZG_CUDA(cudaSetDevice(device));
  size_t free_b = 0, total_b = 0;
  ZG_CUDA(cudaMemGetInfo(&free_b, &total_b));
  if (out->bytes > px_bits_.cap && out->bytes > free_b / 4) {
    *too_big = true;
    return ZG_OK;
  }
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  if (!px_bits_.ensure(std::max<uint64_t>(out->bytes, 4)) || !px_str_.ensure(prefix.size()) || !px_ctrl_.ensure(8)) {
    if (err) *err = "out of device memory (prefix bitmaps)";
    return ZG_ENOMEM;
  }
  const uint64_t uploads = ingress_ ? ingress_->sync_uploads : 0;
  if (int rc = ingress_sync(store, stream, err)) {
    if (rc != ZG_ENOMEM) return rc;
    // the mirror did not fit: the host store answers, as for bitmaps over the budget. A sync that stopped part way
    // leaves the mirror behind the store, so it is dropped and the next call builds it again.
    ingress_reset();
    *too_big = true;
    return ZG_OK;
  }
  st->syncs += ingress_->sync_uploads - uploads;
  PrefixPlan p{};
  p.prefix = px_str_.as<uint8_t>();
  p.len = prefix.size();
  p.matched = px_ctrl_.as<unsigned long long>();
  ZG_CUDA(cudaMemcpyAsync(px_str_.p, prefix.data(), prefix.size(), cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemsetAsync(px_bits_.p, 0, out->bytes, stream));
  ZG_CUDA(cudaMemsetAsync(p.matched, 0, 8, stream));
  std::vector<PrefixType> types;
  uint64_t recs = 0;
  for (size_t t = 0; t < nt; ++t) {
    if (!want[t]) continue;
    out->type[t] = px_bits_.as<uint32_t>() + word0[t];
    if (t >= ingress_->types.size() || ingress_->types[t].host_offs.empty()) continue;  // no interned name
    const IngressMirror::Type& y = ingress_->types[t];
    PrefixType x{};
    x.arena = y.arena.as<uint8_t>();
    x.offs = y.offs.as<unsigned long long>();
    x.n_recs = y.host_offs.size();
    x.bits = px_bits_.as<uint32_t>() + word0[t];
    x.n_ids = out->n_ids[t];
    types.push_back(x);
    recs = std::max<uint64_t>(recs, x.n_recs);
  }
  for (size_t at = 0; at < types.size(); at += kMaxPrefixTypes) {
    p.n_types = static_cast<uint32_t>(std::min<size_t>(kMaxPrefixTypes, types.size() - at));
    std::copy(types.begin() + at, types.begin() + at + p.n_types, p.type);
    for (uint32_t k = 0; k < p.n_types; ++k) st->names += p.type[k].n_recs;
    prefix_match_kernel<<<ingress_grid(recs, sm_count_), kIngressThreads, 0, stream>>>(p);
    ++launches;
    ++st->launches;
  }
  ZG_CUDA(cudaGetLastError());
  unsigned long long matched = 0;
  ZG_CUDA(cudaMemcpyAsync(&matched, p.matched, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  st->matched += matched;
  return ZG_OK;
}

// ---- device ingress ----------------------------------------------------------------------------

IngressMirror::~IngressMirror() {
  for (auto& t : types)
    for (auto* b : {&t.arena, &t.offs, &t.slots}) b->release();
  for (auto* b : {&stage, &items, &out, &one, &bad}) b->release();
  if (pin) cudaFreeHost(pin);
  if (pin_out) cudaFreeHost(pin_out);
}

uint64_t IngressMirror::device_bytes() const {
  uint64_t b = 0;
  for (const auto& t : types) b += t.arena.cap + t.offs.cap + t.slots.cap;
  return b;
}

static unsigned ingress_grid(uint64_t n, int sm_count) {
  const uint64_t want = (n + kIngressThreads - 1) / kIngressThreads;
  return static_cast<unsigned>(std::max<uint64_t>(1, std::min<uint64_t>(want, uint64_t(std::max(sm_count, 1)) * 16)));
}

// Names are appended between schema loads, so the mirror only ever uploads the arena bytes it has not seen. A
// retirement rewrites the arena; zg_retire_unused_names then drops the mirror (ingress_reset) and the next call rebuilds it.
int Device::ingress_sync(const Store& store, cudaStream_t st, std::string* err) {
  constexpr uint64_t kMinTable = 1024;
  if (!ingress_) ingress_.reset(new IngressMirror());
  IngressMirror& m = *ingress_;
  if (m.types.size() != store.n_types()) m.types.resize(store.n_types());
  bool uploaded = false;
  for (size_t t = 0; t < m.types.size(); ++t) {
    const std::vector<char>& ar = store.name_arena(static_cast<int>(t));
    IngressMirror::Type& y = m.types[t];
    if (ar.size() < y.bytes) {  // not the arena this mirror was built from: start the type over
      m.names -= y.host_offs.size();
      for (auto* b : {&y.arena, &y.offs, &y.slots}) b->release();
      y = IngressMirror::Type{};
    }
    if (ar.size() == y.bytes) continue;
    if (ar.size() >= kIngressOffMask) {
      if (err) *err = "interned names of one type exceed 2^40 bytes";
      return ZG_ENOMEM;
    }
    uploaded = true;
    const uint64_t n_old = y.host_offs.size();
    for (uint64_t off = y.bytes; off < ar.size();) {
      uint32_t len;
      std::memcpy(&len, ar.data() + off + 4, 4);
      y.host_offs.push_back(off);
      off += 8 + uint64_t(len);
    }
    const uint64_t n_all = y.host_offs.size();
    // arena: the new bytes, or all of them into a buffer twice the size
    if (ar.size() > y.arena.cap) {
      if (!y.arena.ensure(std::max<size_t>(ar.size(), y.arena.cap * 2))) {
        if (err) *err = "out of device memory (name mirror)";
        return ZG_ENOMEM;
      }
      ZG_CUDA(cudaMemcpyAsync(y.arena.p, ar.data(), ar.size(), cudaMemcpyHostToDevice, st));
    } else {
      ZG_CUDA(cudaMemcpyAsync(y.arena.as<char>() + y.bytes, ar.data() + y.bytes, ar.size() - y.bytes,
                              cudaMemcpyHostToDevice, st));
    }
    // record offsets, likewise
    if (n_all * 8 > y.offs.cap) {
      if (!y.offs.ensure(std::max<size_t>(n_all * 8, y.offs.cap * 2))) {
        if (err) *err = "out of device memory (name mirror)";
        return ZG_ENOMEM;
      }
      ZG_CUDA(cudaMemcpyAsync(y.offs.p, y.host_offs.data(), n_all * 8, cudaMemcpyHostToDevice, st));
    } else {
      ZG_CUDA(cudaMemcpyAsync(y.offs.as<uint64_t>() + n_old, y.host_offs.data() + n_old, (n_all - n_old) * 8,
                              cudaMemcpyHostToDevice, st));
    }
    // table: insert the new records, or every record into a table twice the size when the load would pass 1/2
    uint64_t cap = y.cap ? y.cap : kMinTable;
    while (n_all * 2 > cap) cap *= 2;
    uint64_t from = n_old;
    if (cap != y.cap) {
      if (!y.slots.ensure(cap * 8)) {
        if (err) *err = "out of device memory (name mirror)";
        return ZG_ENOMEM;
      }
      ZG_CUDA(cudaMemsetAsync(y.slots.p, 0, cap * 8, st));
      if (y.cap) ++m.rebuilds;
      y.cap = cap;
      from = 0;
    }
    IngressInsertParams p{};
    p.arena = y.arena.as<uint8_t>();
    p.offs = y.offs.as<unsigned long long>();
    p.from = from;
    p.to = n_all;
    p.slots = y.slots.as<unsigned long long>();
    p.mask = cap - 1;
    ingress_insert_kernel<<<ingress_grid(n_all - from, sm_count_), kIngressThreads, 0, st>>>(p);
    ZG_CUDA(cudaGetLastError());
    ++launches;
    y.bytes = ar.size();
    m.names += n_all - n_old;
  }
  if (uploaded) ++m.sync_uploads;
  return ZG_OK;
}

int Device::ingress_resolve(const Store& store, const IngressLiterals& lit, const char* d_res_ids, const uint32_t* d_res_off,
                            const char* d_subj_ids, const uint32_t* d_subj_off, uint64_t n, zg_check* d_out, cudaStream_t st,
                            std::string* err) {
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  int rc = ingress_sync(store, st, err);
  if (rc) return rc;
  IngressMirror& m = *ingress_;
  if (!m.bad.ensure(4) || (lit.one_subj && !m.one.ensure(lit.one_len + 1))) {
    if (err) *err = "out of device memory (ingress scratch)";
    return ZG_ENOMEM;
  }
  ZG_CUDA(cudaMemsetAsync(m.bad.p, 0, 4, st));
  if (lit.one_subj && lit.one_len)
    ZG_CUDA(cudaMemcpyAsync(m.one.p, lit.one_subj, lit.one_len, cudaMemcpyHostToDevice, st));
  auto table = [&](int t) {
    IngressTable x{nullptr, nullptr, 0};
    if (t >= 0 && t < static_cast<int>(m.types.size()) && m.types[t].cap) {
      x.arena = m.types[t].arena.as<uint8_t>();
      x.slots = m.types[t].slots.as<unsigned long long>();
      x.mask = m.types[t].cap - 1;
    }
    return x;
  };
  IngressResolveParams p{};
  p.rt = table(lit.rt);
  p.st = table(lit.st);
  p.res_ids = reinterpret_cast<const uint8_t*>(d_res_ids);
  p.res_off = d_res_off;
  p.subj_ids = lit.one_subj ? m.one.as<uint8_t>() : reinterpret_cast<const uint8_t*>(d_subj_ids);
  p.subj_off = lit.one_subj ? nullptr : d_subj_off;
  p.one_len = lit.one_len;
  p.one_su = lit.one_su;
  p.ok = lit.ok ? 1 : 0;
  p.same_type = lit.rt == lit.st ? 1 : 0;
  p.base = lit.base;
  p.n = n;
  p.tag_mask = kIngressTagMask;
  p.out = d_out;
  p.bad = m.bad.as<unsigned>();
  ingress_resolve_kernel<<<ingress_grid(n, sm_count_), kIngressThreads, 0, st>>>(p);
  ZG_CUDA(cudaGetLastError());
  ++launches;
  unsigned bad = 0;
  ZG_CUDA(cudaMemcpyAsync(&bad, m.bad.p, 4, cudaMemcpyDeviceToHost, st));
  ZG_CUDA(cudaStreamSynchronize(st));
  m.items_resolved += n;
  if (bad) {
    if (err) *err = "offsets must not decrease";
    return ZG_EINVAL;
  }
  return ZG_OK;
}

int Device::ingress_check_host(const Store& store, const IngressLiterals& lit, const char* res_ids, const uint32_t* res_off,
                               const char* subj_ids, const uint32_t* subj_off, uint64_t n, uint8_t* out, std::string* err) {
  if (n == 0) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  for (uint64_t i = 0; i < n; ++i)
    if (res_off[i] > res_off[i + 1] || (subj_off && subj_off[i] > subj_off[i + 1])) {
      if (err) *err = "offsets must not decrease";
      return ZG_EINVAL;
    }
  // one staging area, one copy: [res_off][subj_off][res blob][subj blob], each part 16-byte aligned
  auto al = [](uint64_t b) { return (b + 15) & ~uint64_t(15); };
  const uint64_t off_bytes = (n + 1) * 4, rblob = res_off[n], sblob = subj_off ? subj_off[n] : 0;
  const uint64_t o_soff = al(off_bytes), o_rids = o_soff + (subj_off ? al(off_bytes) : 0), o_sids = o_rids + al(rblob);
  const uint64_t total = o_sids + al(sblob);
  if (!ingress_) ingress_.reset(new IngressMirror());
  IngressMirror& m = *ingress_;
  if (total > m.pin_cap) {
    if (m.pin) cudaFreeHost(m.pin);
    m.pin = nullptr;
    m.pin_cap = 0;
    ZG_CUDA(cudaHostAlloc(&m.pin, total + total / 4, cudaHostAllocDefault));
    m.pin_cap = total + total / 4;
  }
  if (n > m.pin_out_cap) {
    if (m.pin_out) cudaFreeHost(m.pin_out);
    m.pin_out = nullptr;
    m.pin_out_cap = 0;
    ZG_CUDA(cudaHostAlloc(&m.pin_out, n + n / 4, cudaHostAllocDefault));
    m.pin_out_cap = n + n / 4;
  }
  if (!m.stage.ensure(total) || !m.items.ensure(n * sizeof(zg_check)) || !m.out.ensure(n)) {
    if (err) *err = "out of device memory (ingress staging)";
    return ZG_ENOMEM;
  }
  char* pin = static_cast<char*>(m.pin);
  std::memcpy(pin, res_off, off_bytes);
  if (subj_off) std::memcpy(pin + o_soff, subj_off, off_bytes);
  std::memcpy(pin + o_rids, res_ids, rblob);
  if (subj_off) std::memcpy(pin + o_sids, subj_ids, sblob);
  ZG_CUDA(cudaMemcpyAsync(m.stage.p, pin, total, cudaMemcpyHostToDevice, stream));
  char* d = m.stage.as<char>();
  int rc = ingress_resolve(store, lit, d + o_rids, reinterpret_cast<const uint32_t*>(d),
                           subj_off ? d + o_sids : nullptr, subj_off ? reinterpret_cast<const uint32_t*>(d + o_soff) : nullptr,
                           n, m.items.as<zg_check>(), stream, err);
  if (rc) return rc;
  rc = check_device(m.items.as<zg_check>(), n, m.out.as<uint8_t>(), stream, true, nullptr, err);
  if (rc) return rc;
  ZG_CUDA(cudaMemcpyAsync(m.pin_out, m.out.p, n, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  std::memcpy(out, m.pin_out, n);
  return ZG_OK;
}

// ---- zg_import_relationships -----------------------------------------------------------------------

static unsigned import_grid(uint64_t n, int sm_count) {
  const uint64_t want = (n + kImportThreads - 1) / kImportThreads;
  return static_cast<unsigned>(std::max<uint64_t>(1, std::min<uint64_t>(want, uint64_t(std::max(sm_count, 1)) * 16)));
}

int Device::import_check(const Store& store, const std::vector<ImportGroup>& groups, uint64_t n,
                         const std::vector<uint32_t>& extent, bool locate, ImportCheck* out, std::string* err) {
  ZG_CUDA(cudaSetDevice(device));
  *out = ImportCheck{};
  out->type_count.assign(extent.size(), 0);
  if (!import_) import_.reset(new ImportScratch());
  ImportScratch& x = *import_;
  x.n = n;
  x.n_groups = static_cast<uint32_t>(groups.size());
  if (n == 0) return ZG_OK;
  int rc = ingress_sync(store, stream, err);
  if (rc) return rc;
  auto need = [&](DevBuf& b, size_t bytes) {
    if (b.ensure(bytes)) return true;
    if (err) *err = "out of device memory (import scratch)";
    return false;
  };
  // stage: every group's blobs and offsets (res_off then subj_off), and the groups
  std::shared_ptr<Snapshot> snap_now = snap;
  std::vector<ImportGroupDev> gd(groups.size());
  uint64_t blob_bytes = 0, off_words = 0;
  for (size_t g = 0; g < groups.size(); ++g) {
    const ImportGroup& h = groups[g];
    ImportGroupDev& d = gd[g];
    d.item0 = h.item0;
    d.n = h.n;
    d.res_blob = blob_bytes;
    blob_bytes += h.res_off[h.n];
    d.subj_blob = blob_bytes;
    blob_bytes += h.subj_off[h.n];
    d.off0 = off_words;
    off_words += 2 * (h.n + 1);
    d.rtype = h.rtype;
    d.stype = h.stype;
    d.rel = h.rel;
    d.srel = h.srel;
    d.pos_plain = h.pos_plain;
    d.pos_wild = h.pos_wild;
    d.k_plain = h.k_plain;
    d.k_wild = h.k_wild;
    if (snap_now && h.rel_index < snap_now->rels.size()) {
      const DRel& r = snap_now->rels[h.rel_index];
      d.row_base = r.row_base;
      d.stride = r.stride;
      d.nres = r.nres;
    }
  }
  const uint64_t occ = 2 * n;
  uint64_t cap = 64;
  while (cap < 2 * occ) cap *= 2;
  const size_t nt = extent.size();
  if (!need(x.groups, gd.size() * sizeof(ImportGroupDev)) || !need(x.blob, blob_bytes + 8) || !need(x.offs, off_words * 4) ||
      !need(x.tables, nt * sizeof(IngressTable)) || !need(x.slots, cap * 8) || !need(x.first, cap * 8) ||
      !need(x.hash, cap * 8) || !need(x.slot_type, cap * 4) || !need(x.occ_id, occ * 4) || !need(x.occ_slot, occ * 4) ||
      !need(x.ctrl, 4 * 8) || !need(x.extent, nt * 4) || !need(x.type_start, nt * 8))
    return ZG_ENOMEM;
  for (size_t g = 0; g < groups.size(); ++g) {
    const ImportGroup& h = groups[g];
    ZG_CUDA(cudaMemcpyAsync(x.blob.as<char>() + gd[g].res_blob, h.res_ids, h.res_off[h.n], cudaMemcpyHostToDevice, stream));
    ZG_CUDA(cudaMemcpyAsync(x.blob.as<char>() + gd[g].subj_blob, h.subj_ids, h.subj_off[h.n], cudaMemcpyHostToDevice, stream));
    ZG_CUDA(cudaMemcpyAsync(x.offs.as<uint32_t>() + gd[g].off0, h.res_off, (h.n + 1) * 4, cudaMemcpyHostToDevice, stream));
    ZG_CUDA(cudaMemcpyAsync(x.offs.as<uint32_t>() + gd[g].off0 + h.n + 1, h.subj_off, (h.n + 1) * 4, cudaMemcpyHostToDevice,
                            stream));
  }
  ZG_CUDA(cudaMemcpyAsync(x.groups.p, gd.data(), gd.size() * sizeof(ImportGroupDev), cudaMemcpyHostToDevice, stream));
  std::vector<IngressTable> tabs(nt, IngressTable{nullptr, nullptr, 0});
  for (size_t t = 0; t < nt && t < ingress_->types.size(); ++t)
    if (ingress_->types[t].cap) {
      tabs[t].arena = ingress_->types[t].arena.as<uint8_t>();
      tabs[t].slots = ingress_->types[t].slots.as<unsigned long long>();
      tabs[t].mask = ingress_->types[t].cap - 1;
    }
  ZG_CUDA(cudaMemcpyAsync(x.tables.p, tabs.data(), nt * sizeof(IngressTable), cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemcpyAsync(x.extent.p, extent.data(), nt * 4, cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemsetAsync(x.slots.p, 0, cap * 8, stream));
  ZG_CUDA(cudaMemsetAsync(x.first.p, 0xFF, cap * 8, stream));
  ZG_CUDA(cudaMemsetAsync(x.ctrl.p, 0xFF, 2 * 8, stream));
  ZG_CUDA(cudaMemsetAsync(x.ctrl.as<unsigned long long>() + 2, 0, 2 * 8, stream));
  unsigned long long* ctrl = x.ctrl.as<unsigned long long>();
  ImportCall call{x.groups.as<ImportGroupDev>(), x.n_groups, x.blob.as<uint8_t>(), x.offs.as<uint32_t>(), n};
  cudaEvent_t ev[4];
  for (auto& e : ev) ZG_CUDA(cudaEventCreate(&e));
  struct Events {
    cudaEvent_t* e;
    ~Events() {
      for (int i = 0; i < 4; ++i) cudaEventDestroy(e[i]);
    }
  } ev_guard{ev};
  ZG_CUDA(cudaEventRecord(ev[0], stream));

  // 1. names
  ImportNamesParams np{};
  np.c = call;
  np.tables = x.tables.as<IngressTable>();
  np.slots = x.slots.as<unsigned long long>();
  np.mask = cap - 1;
  np.first = x.first.as<unsigned long long>();
  np.hash = x.hash.as<unsigned long long>();
  np.slot_type = x.slot_type.as<uint32_t>();
  np.occ_id = x.occ_id.as<uint32_t>();
  np.occ_slot = x.occ_slot.as<uint32_t>();
  np.bad = ctrl;
  np.tag_mask = kIngressTagMask;
  np.found = ctrl + 2;
  import_names_kernel<<<import_grid(occ, sm_count_), kImportThreads, 0, stream>>>(np);
  ZG_CUDA(cudaGetLastError());
  ++launches;

  // 2. new names sorted by (type, first occurrence); the host needs each type's first rank for the temporary ids
  uint64_t n_new = 0;
  {
    if (!need(x.new_keys, cap * 8) || !need(x.new_vals, cap * 4)) return ZG_ENOMEM;
    import_compact_kernel<<<import_grid(cap, sm_count_), kImportThreads, 0, stream>>>(
        x.slots.as<unsigned long long>(), cap, x.first.as<unsigned long long>(), x.slot_type.as<uint32_t>(),
        x.new_keys.as<unsigned long long>(), x.new_vals.as<uint32_t>(), ctrl + 3);
    ZG_CUDA(cudaGetLastError());
    ++launches;
    unsigned long long h[4];
    ZG_CUDA(cudaMemcpyAsync(h, ctrl, sizeof(h), cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    out->bad = h[0];
    out->found = h[2];
    n_new = h[3];
  }
  ZG_CUDA(cudaEventRecord(ev[1], stream));
  if (n_new) {
    if (!need(x.new_keys2, n_new * 8) || !need(x.new_vals2, n_new * 4) || !need(x.slot_tmp, cap * 4) ||
        !need(x.out_hash, n_new * 8))
      return ZG_ENOMEM;
    size_t tmp = 0;
    int end_bit = 48;
    while ((uint64_t(1) << (end_bit - 48)) < nt) ++end_bit;
    ZG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, x.new_keys.as<unsigned long long>(), x.new_keys2.as<unsigned long long>(),
                                            x.new_vals.as<uint32_t>(), x.new_vals2.as<uint32_t>(), n_new, 0, end_bit, stream));
    if (!need(x.cub, tmp)) return ZG_ENOMEM;
    ZG_CUDA(cub::DeviceRadixSort::SortPairs(x.cub.p, tmp, x.new_keys.as<unsigned long long>(), x.new_keys2.as<unsigned long long>(),
                                            x.new_vals.as<uint32_t>(), x.new_vals2.as<uint32_t>(), n_new, 0, end_bit, stream));
    out->new_keys.resize(n_new);
    ZG_CUDA(cudaMemcpyAsync(out->new_keys.data(), x.new_keys2.p, n_new * 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    std::vector<uint64_t> start(nt, 0);
    for (uint64_t j = n_new; j-- > 0;) {
      const uint32_t t = static_cast<uint32_t>(out->new_keys[j] >> 48);
      start[t] = j;
      ++out->type_count[t];
    }
    ZG_CUDA(cudaMemcpyAsync(x.type_start.p, start.data(), nt * 8, cudaMemcpyHostToDevice, stream));
    import_rank_kernel<<<import_grid(n_new, sm_count_), kImportThreads, 0, stream>>>(
        x.new_keys2.as<unsigned long long>(), x.new_vals2.as<uint32_t>(), n_new, x.extent.as<uint32_t>(),
        x.type_start.as<unsigned long long>(), x.hash.as<unsigned long long>(), x.slot_tmp.as<uint32_t>(),
        x.out_hash.as<unsigned long long>());
    ZG_CUDA(cudaGetLastError());
    ++launches;
    out->new_hash.resize(n_new);
    ZG_CUDA(cudaMemcpyAsync(out->new_hash.data(), x.out_hash.p, n_new * 8, cudaMemcpyDeviceToHost, stream));
  }

  // 3. tuples and keys, sorted stably by K (low word, then high word)
  if (!need(x.tuples, n * sizeof(zg_tuple)) || !need(x.key_hi, n * 8) || !need(x.key_lo, n * 8) || !need(x.key_hi2, n * 8) ||
      !need(x.key_lo2, n * 8) || !need(x.vals, n * 4) || !need(x.vals2, n * 4) || !need(x.known, n) || !need(x.slot_tmp, 4))
    return ZG_ENOMEM;
  ImportAssembleParams ap{};
  ap.c = call;
  ap.occ_id = x.occ_id.as<uint32_t>();
  ap.occ_slot = x.occ_slot.as<uint32_t>();
  ap.slot_tmp = x.slot_tmp.as<uint32_t>();
  ap.tuples = x.tuples.as<zg_tuple>();
  ap.key_hi = x.key_hi.as<unsigned long long>();
  ap.key_lo = x.key_lo.as<unsigned long long>();
  ap.vals = x.vals.as<uint32_t>();
  ap.known = x.known.as<uint8_t>();
  import_assemble_kernel<<<import_grid(n, sm_count_), kImportThreads, 0, stream>>>(ap);
  ZG_CUDA(cudaGetLastError());
  ++launches;
  {
    // two stable passes: by the low words, then by the high words gathered into that order; equal keys keep call order
    size_t t1 = 0, t2 = 0;
    ZG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t1, x.key_lo.as<unsigned long long>(), x.key_lo2.as<unsigned long long>(),
                                            x.vals.as<uint32_t>(), x.vals2.as<uint32_t>(), n, 0, 64, stream));
    ZG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t2, x.key_hi2.as<unsigned long long>(), x.key_lo2.as<unsigned long long>(),
                                            x.vals2.as<uint32_t>(), x.vals.as<uint32_t>(), n, 0, 64, stream));
    if (!need(x.cub, std::max(t1, t2))) return ZG_ENOMEM;
    ZG_CUDA(cub::DeviceRadixSort::SortPairs(x.cub.p, t1, x.key_lo.as<unsigned long long>(), x.key_lo2.as<unsigned long long>(),
                                            x.vals.as<uint32_t>(), x.vals2.as<uint32_t>(), n, 0, 64, stream));
    import_gather_kernel<<<import_grid(n, sm_count_), kImportThreads, 0, stream>>>(
        x.key_hi.as<unsigned long long>(), x.vals2.as<uint32_t>(), n, x.key_hi2.as<unsigned long long>());
    ZG_CUDA(cudaGetLastError());
    ++launches;
    ZG_CUDA(cub::DeviceRadixSort::SortPairs(x.cub.p, t2, x.key_hi2.as<unsigned long long>(), x.key_lo2.as<unsigned long long>(),
                                            x.vals2.as<uint32_t>(), x.vals.as<uint32_t>(), n, 0, 64, stream));
  }
  ZG_CUDA(cudaEventRecord(ev[2], stream));

  // 4. duplicates: equal neighbours in K order, and the items the resident snapshot holds
  import_adjacent_kernel<<<import_grid(n, sm_count_), kImportThreads, 0, stream>>>(
      x.key_hi.as<unsigned long long>(), x.key_lo.as<unsigned long long>(), x.vals.as<uint32_t>(), n, ctrl + 1);
  ZG_CUDA(cudaGetLastError());
  ++launches;
  if (locate && snap_now) {
    ImportLocateParams lp{};
    lp.c = call;
    lp.tuples = x.tuples.as<zg_tuple>();
    lp.known = x.known.as<uint8_t>();
    lp.row_ptr = snap_now->row_ptr.as<uint32_t>();
    lp.col = snap_now->col.as<uint32_t>();
    lp.owner_rank = 0;
    lp.owner_count = 1;
    lp.dup = ctrl + 1;
    import_locate_kernel<<<import_grid(n, sm_count_), kImportThreads, 0, stream>>>(lp);
    ZG_CUDA(cudaGetLastError());
    ++launches;
  }
  ZG_CUDA(cudaEventRecord(ev[3], stream));
  unsigned long long dup = 0;
  ZG_CUDA(cudaMemcpyAsync(&dup, ctrl + 1, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  out->dup = dup;
  float a = 0, b = 0, c = 0;
  cudaEventElapsedTime(&a, ev[0], ev[1]);
  cudaEventElapsedTime(&b, ev[1], ev[2]);
  cudaEventElapsedTime(&c, ev[2], ev[3]);
  out->ms_names = a;
  out->ms_sort = b;
  out->ms_dups = c;
  return ZG_OK;
}

void Device::import_release() {
  if (!import_) return;
  cudaSetDevice(device);
  import_.reset();
}

int Device::import_locate(const Device& src, uint64_t* dup, std::string* err) {
  *dup = ~0ull;
  const ImportScratch* x = src.import_.get();
  std::shared_ptr<Snapshot> s = snap;
  if (!x || !x->n || !s) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (!import_) import_.reset(new ImportScratch());
  if (!import_->ctrl.ensure(8)) {
    if (err) *err = "out of device memory (import scratch)";
    return ZG_ENOMEM;
  }
  unsigned long long* d = import_->ctrl.as<unsigned long long>();
  ZG_CUDA(cudaMemsetAsync(d, 0xFF, 8, stream));
  ImportLocateParams lp{};
  lp.c = ImportCall{x->groups.as<ImportGroupDev>(), x->n_groups, x->blob.as<uint8_t>(), x->offs.as<uint32_t>(), x->n};
  lp.tuples = x->tuples.as<zg_tuple>();
  lp.known = x->known.as<uint8_t>();
  lp.row_ptr = s->row_ptr.as<uint32_t>();
  lp.col = s->col.as<uint32_t>();
  lp.owner_rank = own_rank;
  lp.owner_count = own_count;
  lp.dup = d;
  import_locate_kernel<<<import_grid(x->n, sm_count_), kImportThreads, 0, stream>>>(lp);
  ZG_CUDA(cudaGetLastError());
  ++launches;
  unsigned long long h = 0;
  ZG_CUDA(cudaMemcpyAsync(&h, d, 8, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  *dup = h;
  return ZG_OK;
}

int Device::import_finish(const std::vector<uint32_t>& ids, const std::vector<uint64_t>& base,
                          const std::vector<uint32_t>& rtype_of_rel, std::vector<zg_tuple>* tuples, std::string* err) {
  ZG_CUDA(cudaSetDevice(device));
  ImportScratch& x = *import_;
  tuples->resize(x.n);
  if (!x.n) return ZG_OK;
  if (!x.ids.ensure(std::max<size_t>(ids.size(), 1) * 4) || !x.base.ensure(base.size() * 8) ||
      !x.rtype_of_rel.ensure(rtype_of_rel.size() * 4)) {
    if (err) *err = "out of device memory (import scratch)";
    return ZG_ENOMEM;
  }
  if (!ids.empty()) ZG_CUDA(cudaMemcpyAsync(x.ids.p, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemcpyAsync(x.base.p, base.data(), base.size() * 8, cudaMemcpyHostToDevice, stream));
  ZG_CUDA(cudaMemcpyAsync(x.rtype_of_rel.p, rtype_of_rel.data(), rtype_of_rel.size() * 4, cudaMemcpyHostToDevice, stream));
  import_remap_kernel<<<import_grid(x.n, sm_count_), kImportThreads, 0, stream>>>(
      x.tuples.as<zg_tuple>(), x.n, x.rtype_of_rel.as<uint32_t>(), x.extent.as<uint32_t>(), x.base.as<unsigned long long>(),
      x.ids.as<uint32_t>());
  ZG_CUDA(cudaGetLastError());
  ++launches;
  ZG_CUDA(cudaMemcpyAsync(tuples->data(), x.tuples.p, x.n * sizeof(zg_tuple), cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  return ZG_OK;
}

int Device::expand(const std::vector<ExpandReq>& reqs, uint64_t cap, std::vector<zg_expand_node>* nodes,
                   std::vector<zg_expand_subject>* subjects, std::vector<int32_t>* status, std::string* err) {
  nodes->clear();
  subjects->clear();
  status->assign(reqs.size(), ZG_OK);
  x_last_ms.clear();
  std::shared_ptr<Snapshot> s = snap;
  if (!s) {
    if (err) *err = "no snapshot published";
    return ZG_ENOSNAPSHOT;
  }
  if (reqs.empty()) return ZG_OK;
  ZG_CUDA(cudaSetDevice(device));
  if (have_last_) ZG_CUDA(cudaStreamWaitEvent(stream, last_done_, 0));
  // An Expand is a rare debugging call whose output can be large: its scratch is freed when it returns.
  struct Scratch {
    DevBuf jobs[2], failed, cnt, off, cub, nodes, subj, mask;
    std::vector<cudaEvent_t> ev;
    ~Scratch() {
      for (DevBuf* b : {&jobs[0], &jobs[1], &failed, &cnt, &off, &cub, &nodes, &subj, &mask}) b->release();
      for (cudaEvent_t e : ev) cudaEventDestroy(e);
    }
  } x;
  auto oom = [&](const char* what) {
    if (err) *err = std::string("out of device memory (ExpandPermissionTree ") + what + ")";
    return ZG_ENOMEM;
  };
  // grows b to `want` bytes, keeping its first `used`
  auto grow = [&](DevBuf& b, size_t used, size_t want) -> bool {
    if (want <= b.cap) return true;
    DevBuf nb;
    if (!nb.ensure(std::max(want, b.cap * 2))) return false;
    if (used && cudaMemcpyAsync(nb.p, b.p, used, cudaMemcpyDeviceToDevice, stream) != cudaSuccess) {
      nb.release();
      return false;
    }
    b.release();  // cudaFree waits for the copy
    b = nb;
    return true;
  };
  const uint64_t R = reqs.size();
  unsigned long long mask = 0;  // bit c: a job of the level has a template of c counted nodes
  {
    std::vector<XJob> j0(R);
    for (uint64_t i = 0; i < R; ++i) {
      j0[i] = XJob{static_cast<uint32_t>(i), UINT32_MAX, 0, reqs[i].res, reqs[i].tmpl, 0};
      mask |= 1ull << reqs[i].ncount;
    }
    if (!x.jobs[0].ensure(R * sizeof(XJob)) || !x.failed.ensure(R * 4) || !x.mask.ensure(8)) return oom("jobs");
    ZG_CUDA(cudaMemcpyAsync(x.jobs[0].p, j0.data(), R * sizeof(XJob), cudaMemcpyHostToDevice, stream));
    ZG_CUDA(cudaMemsetAsync(x.failed.p, 0, R * 4, stream));
  }
  XParams p{};
  p.row_ptr = s->row_ptr.as<uint32_t>();
  p.col = s->col.as<uint32_t>();
  p.exp = s->exp.p ? s->exp.as<uint32_t>() : nullptr;
  p.rels = s->x_rels.as<DRel>();
  p.cls = s->x_cls.as<DCls>();
  p.nodes = s->x_nodes.as<XNode>();
  p.tgts = s->x_tgts.as<uint32_t>();
  p.counted = s->x_counted.as<uint32_t>();
  p.now = now;
  p.failed = x.failed.as<uint32_t>();
  p.next_mask = x.mask.as<unsigned long long>();
  auto over_cap = [&]() {
    if (err)
      *err = "ExpandPermissionTree: the trees pass " + std::to_string(cap) +
             " nodes plus subjects (ZGPU_EXPAND_CAP); expand fewer or smaller trees per call";
    return ZG_ENOMEM;
  };
  uint64_t n_jobs = R, n_nodes = 0, n_subj = 0, levels = 0;
  int cur = 0;
  while (n_jobs) {
    p.m = expand_warps(mask);
    // every (job, counted node) is a node of the output: the level's scratch stays within the cap's size
    if (n_nodes + n_subj + n_jobs * p.m > cap) return over_cap();
    const uint64_t n = n_jobs * p.m;
    if (!x.cnt.ensure((3 * n + 1) * 8) || !x.off.ensure((3 * n + 1) * 8)) return oom("counts");
    unsigned long long* cnt = x.cnt.as<unsigned long long>();
    unsigned long long* off = x.off.as<unsigned long long>();
    size_t tb = 0;
    ZG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, off, 3 * n + 1, stream));
    if (!x.cub.ensure(tb)) return oom("scan");
    while (x.ev.size() < 5 * (levels + 1)) {  // count, scan, emit: begin and end (emit after the allocations)
      cudaEvent_t e;
      ZG_CUDA(cudaEventCreate(&e));
      x.ev.push_back(e);
    }
    cudaEvent_t* ev = x.ev.data() + 5 * levels;
    ZG_CUDA(cudaMemsetAsync(cnt + 3 * n, 0, 8, stream));
    p.jobs = x.jobs[cur].as<XJob>();
    p.n_jobs = n_jobs;
    p.cnt = cnt;
    p.off = off;
    const unsigned blocks = static_cast<unsigned>((n * 32 + kExpandThreads - 1) / kExpandThreads);
    ZG_CUDA(cudaEventRecord(ev[0], stream));
    expand_count_kernel<<<blocks, kExpandThreads, 0, stream>>>(p);
    ZG_CUDA(cudaGetLastError());
    ZG_CUDA(cudaEventRecord(ev[1], stream));
    ZG_CUDA(cub::DeviceScan::ExclusiveSum(x.cub.p, tb, cnt, off, 3 * n + 1, stream));
    ZG_CUDA(cudaEventRecord(ev[2], stream));
    unsigned long long tot[3];
    for (int i = 0; i < 3; ++i)
      ZG_CUDA(cudaMemcpyAsync(tot + i, off + (i + 1) * n, 8, cudaMemcpyDeviceToHost, stream));
    ZG_CUDA(cudaStreamSynchronize(stream));
    const uint64_t lvl_nodes = tot[0], lvl_subj = tot[1] - tot[0], next = tot[2] - tot[1];
    // each next-level job is at least one node
    if (n_nodes + lvl_nodes + n_subj + lvl_subj + next > cap) return over_cap();
    if (!grow(x.nodes, n_nodes * sizeof(zg_expand_node), (n_nodes + lvl_nodes) * sizeof(zg_expand_node)) ||
        !grow(x.subj, n_subj * sizeof(zg_expand_subject), (n_subj + lvl_subj) * sizeof(zg_expand_subject)) ||
        !x.jobs[cur ^ 1].ensure(next * sizeof(XJob)))
      return oom("output");
    p.node_base = n_nodes;
    p.subj_base = n_subj;
    p.out_nodes = x.nodes.as<zg_expand_node>();
    p.out_subj = x.subj.as<zg_expand_subject>();
    p.next = x.jobs[cur ^ 1].as<XJob>();
    ZG_CUDA(cudaMemsetAsync(p.next_mask, 0, 8, stream));
    ZG_CUDA(cudaEventRecord(ev[3], stream));
    expand_emit_kernel<<<blocks, kExpandThreads, 0, stream>>>(p);
    ZG_CUDA(cudaGetLastError());
    ZG_CUDA(cudaEventRecord(ev[4], stream));
    if (next) {
      ZG_CUDA(cudaMemcpyAsync(&mask, p.next_mask, 8, cudaMemcpyDeviceToHost, stream));
      ZG_CUDA(cudaStreamSynchronize(stream));
    }
    launches += 2;
    n_nodes += lvl_nodes;
    n_subj += lvl_subj;
    n_jobs = next;
    cur ^= 1;
    ++levels;
  }
  std::vector<uint32_t> failed(R);
  nodes->resize(n_nodes);
  subjects->resize(n_subj);
  if (n_nodes) ZG_CUDA(cudaMemcpyAsync(nodes->data(), x.nodes.p, n_nodes * sizeof(zg_expand_node), cudaMemcpyDeviceToHost, stream));
  if (n_subj) ZG_CUDA(cudaMemcpyAsync(subjects->data(), x.subj.p, n_subj * sizeof(zg_expand_subject), cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaMemcpyAsync(failed.data(), x.failed.p, R * 4, cudaMemcpyDeviceToHost, stream));
  ZG_CUDA(cudaStreamSynchronize(stream));
  for (uint64_t l = 0; l < levels; ++l)
    for (int i : {0, 1, 3}) {
      float ms = 0;
      cudaEventElapsedTime(&ms, x.ev[5 * l + i], x.ev[5 * l + i + 1]);
      x_last_ms.push_back(ms);
    }
  bool any_failed = false;
  for (uint64_t i = 0; i < R; ++i)
    if (failed[i]) {
      (*status)[i] = ZG_EDEPTH;
      any_failed = true;
    }
  if (any_failed) expand_drop_failed(failed, nodes, subjects);
  for (uint64_t i = 0; i < R; ++i) x_trees += failed[i] ? 0 : 1;
  x_levels += levels;
  x_nodes_out += nodes->size();
  x_subjects_out += subjects->size();
  return ZG_OK;
}

}  // namespace zg
