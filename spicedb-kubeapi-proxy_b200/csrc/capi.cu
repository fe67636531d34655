// capi.cu -- the C ABI declared in include/zgpu.h. Thin glue: argument checks,
// string <-> id resolution, locking; the work is in store.cc and device.cu.
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <deque>
#include <functional>
#include <memory>
#include <atomic>
#include <mutex>
#include <shared_mutex>
#include <new>
#include <string>
#include <string_view>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/zgpu.h"
#include "closure_sig.cuh"
#include "device.h"
#include "schema.h"
#include "store.h"

using namespace zg;

// The device lock is FIFO. std::mutex makes no fairness promise, and glibc's lets a thread that unlocks and locks again
// at once overtake every sleeper: a caller issuing writes back to back (each publishes under this lock) starved the
// leaders of the check and lookup queues for seconds in tests/cabi/batcher_stress.c. Few threads ever wait here (one
// leader per queue, writers, direct callers), so one shared condition variable is enough.
class FairMutex {
  std::mutex m_;
  std::condition_variable cv_;
  uint64_t next_ = 0, serving_ = 0;

 public:
  void lock() {
    std::unique_lock<std::mutex> lk(m_);
    const uint64_t ticket = next_++;
    cv_.wait(lk, [&] { return serving_ == ticket; });
  }
  void unlock() {
    {
      std::lock_guard<std::mutex> lk(m_);
      ++serving_;
    }
    cv_.notify_all();
  }
};

// A caller's place in a GroupQueue, and its result.
struct QueuedJob {
  int rc = ZG_OK;
  std::string err;
  bool done = false, lead = false;
  std::condition_variable cv;  // every waiter sleeps on its own: a finished group wakes exactly its members and
                               // ONE next leader, not every queued caller (1 000 of them under BASELINE config 5)
};

// Coalescing queue ("group commit") for zg_check_bulk and LookupResources. The proxy calls the boundary from one
// goroutine per rule check (pkg/authz/check.go:77-93) and per list request (pkg/authz/postfilter.go:127-134): many
// concurrent, mostly small calls. The first caller to arrive becomes the leader; while its group runs later callers
// queue, and the next leader answers ALL of them (as many as one group takes) with one launch sequence. No timer:
// batching is driven purely by arrivals during the previous group. Job derives from QueuedJob.
template <class Job>
class GroupQueue {
  std::mutex m_;
  std::vector<Job*> queue_;
  bool leader_active_ = false;

 public:
  uint64_t groups = 0, waited = 0, handed_over = 0;  // protocol counters

  // Queues `me` and returns once a group holding it has run. take(queue) = how many jobs from the front of the queue
  // one group takes (at least one); run(group) answers them under the device lock and sets each job's rc / err.
  template <class Take, class Run>
  void submit(Job* me, FairMutex& device, Take&& take, Run&& run) {
    std::unique_lock<std::mutex> lk(m_);
    queue_.push_back(me);
    if (leader_active_) {
      ++waited;
      me->cv.wait(lk, [&] { return me->done || me->lead; });
    }
    if (me->done) return;
    // leader (nobody was leading, or the previous leader handed over to the head of the queue -- me): take as many
    // queued jobs as one group takes, mine first, answer them, wake their callers, hand leadership on
    leader_active_ = true;
    std::vector<Job*> group;
    lk.unlock();
    {
      // the device first, the group second: whatever queued while this leader waited for the GPU (behind another
      // queue's group, a publish, the previous group's tail) rides along
      std::lock_guard<FairMutex> dev_lock(device);
      lk.lock();
      const auto n = static_cast<long>(take(queue_));
      group.assign(queue_.begin(), queue_.begin() + n);
      queue_.erase(queue_.begin(), queue_.begin() + n);
      lk.unlock();
      run(group);
    }
    lk.lock();
    ++groups;
    for (Job* j : group) {
      j->done = true;
      if (j != me) j->cv.notify_one();
    }
    if (!queue_.empty()) {
      ++handed_over;
      queue_.front()->lead = true;
      queue_.front()->cv.notify_one();
    } else {
      leader_active_ = false;
    }
  }
};

// One zg_check_bulk call.
struct BatchReq : QueuedJob {
  const zg_check* items = nullptr;
  uint64_t n = 0;
  uint8_t* out = nullptr;
};
static constexpr uint64_t kMaxItemsPerLaunch = 1ull << 24;  // of a check group (one caller's items are never split)

// One engine may own several GPUs of the box (zg_config.n_devices): every device holds a REPLICA of the
// snapshot (1e8 relationships = 2 GB, two orders of magnitude under one GPU's HBM) and answers its slice of
// every batch; no data-path collective (SURVEY.md 8e mode 1). Device 0 is driven inline by the calling
// thread, every further device by its own worker thread (CUDA's current device is per-thread state).
struct DeviceWorker {
  std::thread th;
  std::mutex m;
  std::condition_variable cv;
  std::function<void()> task;
  bool has = false, stop = false, busy = false;
  void start() {
    th = std::thread([this] {
      std::unique_lock<std::mutex> lk(m);
      for (;;) {
        cv.wait(lk, [this] { return has || stop; });
        if (stop) return;
        std::function<void()> f = std::move(task);
        has = false;
        lk.unlock();
        f();
        lk.lock();
        busy = false;
        cv.notify_all();
      }
    });
  }
  void submit(std::function<void()> f) {
    std::unique_lock<std::mutex> lk(m);
    cv.wait(lk, [this] { return !busy; });
    task = std::move(f);
    has = busy = true;
    cv.notify_all();
  }
  void wait() {
    std::unique_lock<std::mutex> lk(m);
    cv.wait(lk, [this] { return !busy; });
  }
  ~DeviceWorker() {
    if (th.joinable()) {
      {
        std::lock_guard<std::mutex> lk(m);
        stop = true;
      }
      cv.notify_all();
      th.join();
    }
  }
};
struct Replica {
  Device dev;
  DeviceWorker worker;
};
// what one run of the sharded check protocol cost: pass levels, sub-queries the shards raised to each other, and the
// times the host waited for the devices
struct PeerCounts {
  uint64_t levels = 0, subqueries = 0, round_trips = 0;
};

struct zg_engine {
  // Two locks, always taken in this order:
  //   mu     the device: one launch sequence (a coalesced group of checks, a batch of lookups) or one publish at
  //          a time. Held for milliseconds by whoever leads a group.
  //   names  the schema and the store (interning tables, relationship set): shared by everything that resolves
  //          or renders names, exclusive for writers. Never held across GPU work except by a publish, so that
  //          callers can resolve their strings and QUEUE behind a running group instead of waiting for it.
  FairMutex mu;  // the device lock: one launch sequence or publish at a time
  mutable std::shared_mutex names;
  std::vector<std::unique_ptr<Replica>> replicas;  // devices 1 .. n-1 (device 0 is `dev`)
  GroupQueue<BatchReq> batcher;  // zg_check_bulk (ZGPU_BATCHER_STATS=1 prints its counters at destroy)
  Schema schema;
  bool has_schema = false;
  Store store;
  Device dev;
  int64_t clock = 0;
  uint64_t revision = 0;
  std::atomic<bool> dirty{false};  // store changed since the last publish
  bool host_only = false;
  // Concurrent LookupResources calls (one goroutine per list request: pkg/authz/responsefilterer.go:165) are
  // coalesced like the checks: the leader answers up to 64 of them with one batched launch sequence.
  struct LookupKey {
    uint64_t revision = ~0ull;
    uint32_t subj = 0;
    uint16_t res_type = 0, perm = 0, stype = 0, srel = 0;
    int64_t clock = 0;
    bool operator==(const LookupKey& o) const {
      return revision == o.revision && subj == o.subj && res_type == o.res_type && perm == o.perm && stype == o.stype &&
             srel == o.srel && clock == o.clock;
    }
  };
  struct LookupJob : QueuedJob {
    LookupKey key;       // revision / clock filled in by the leader
    bool want_self = false;
    std::vector<uint32_t> ids;
    bool self_member = false;
  };
  GroupQueue<LookupJob> lookups;
  // ZG_E2BIG protocol: recent answers are kept so that a caller's retry with a larger buffer (same arguments,
  // same snapshot revision) does not recompute them. zg_retire_unused_names leaves them valid: every id in an answer is
  // mentioned by a relationship at that revision, and only names no relationship mentions are retired.
  std::deque<std::pair<LookupKey, std::shared_ptr<const std::vector<uint32_t>>>> lookup_cache;
  static constexpr size_t kLookupCache = 128;
  HostSnapshot last_built;  // kept only for zg_debug_row / host-only engines
  bool keep_built = false;
  // Sharded handle (zg_config.n_shards = S > 1): ONE store, S shards of its snapshot. Shard 0 is `dev`, shard k the
  // device of replicas[k - 1] (own_rank k, own_count S); run_sharded drives a check group across them.
  uint32_t n_shards = 1, shard_devices = 1;
  void* group_pin = nullptr;  // a group's items, then its answers (pinned: the shards copy their slices from / to it)
  size_t group_pin_cap = 0;
  PeerCounts last_group;  // zg_stats last_levels / last_subqueries / last_round_trips
  // ZG_FLAG_HANDLE_LOOKUPS: run_sharded_lookup answers LookupResources; zg_handle_lookup_counters
  bool handle_lookups = false;
  uint64_t hl_rounds = 0, hl_levels = 0, hl_round_trips = 0, hl_frontier = 0, hl_candidates = 0, hl_halvings = 0,
           hl_fallbacks = 0;
  // ZG_FLAG_HANDLE_SUBJECTS: run_sharded_subjects answers LookupSubjects; zg_handle_subjects_counters
  bool handle_subjects = false;
  uint64_t hs_lookups = 0, hs_levels = 0, hs_waits = 0, hs_entries = 0, hs_candidates = 0, hs_nowild = 0, hs_fallbacks = 0;
  std::vector<HostSnapshot> shard_built;  // zg_debug_shard_row: the host builder's arrays per shard
  // zg_filter_counters: relationship filters (reads, deletes by filter, preconditions) answered from the snapshot on
  // the device and by Store::match, relationships the device returned, device filters by Device::FilterShape
  std::atomic<uint64_t> flt_device{0}, flt_host{0}, flt_returned{0}, flt_shape[3] = {};
  // zg_page_counters: pages served on the device / by the host store, entries the device windows covered, launches
  std::atomic<uint64_t> pg_device{0}, pg_host{0}, pg_scanned{0}, pg_launches{0};
  // zg_prefix_counters: prefix filters answered on the device / by the host store, names the device scanned, resources
  // it matched, launches of the scans and match lists, names-mirror syncs that uploaded bytes
  std::atomic<uint64_t> px_device{0}, px_host{0}, px_names{0}, px_matched{0}, px_launches{0}, px_syncs{0};
  // zg_lookup_page_counters: LookupResources pages answered by windowed verification / cut from a whole answer (a
  // sharded handle), candidates after the cursor, candidates verified, verification windows
  std::atomic<uint64_t> lp_windowed{0}, lp_cut{0}, lp_after{0}, lp_verified{0}, lp_windows{0};
  uint32_t schema_gen = 0;  // schema loads: a page cursor names the schema it was made under
  // zg_name_counters: names retired by zg_retire_unused_names calls that read the mentions from the snapshots / from
  // the host store (reset with the store by a schema load)
  uint64_t retire_device = 0, retire_host = 0;
  // Bumped by every zg_retire_unused_names call that retires a name, under the device lock and the exclusive names
  // lock, before any freed id can be handed out again (with_stable_names).
  std::atomic<uint64_t> name_epoch{0};
  // zg_debug_set_resolve_hook: called by the string checks and lookups between resolving their names and answering
  // (tests force a retirement and a reuse of the ids into that gap with it); nullptr = none
  void (*resolve_hook)(void*) = nullptr;
  void* resolve_hook_arg = nullptr;
  // zg_import_counters: successful imports on the device / on the host, relationships imported, name occurrences the
  // store had, names interned new; zg_import_last_times: the last successful import's steps, in milliseconds
  uint64_t imp_device = 0, imp_host = 0, imp_rels = 0, imp_found = 0, imp_new = 0;
  double imp_ms[7] = {};
  ~zg_engine() {
    if (group_pin) cudaFreeHost(group_pin);
  }
  // Watch feed (pkg/authz/watch.go:29-31): what WriteRelationships / DeleteRelationships changed,
  // stamped with the revision that made it visible. Bounded: the oldest entries are dropped and
  // a reader that asks for them is told so (as SpiceDB does past its GC window).
  struct WatchEntry {
    uint64_t revision;
    zg_tuple t;
    uint32_t expires_at, op;
  };
  std::deque<WatchEntry> watch_log;
  uint64_t watch_floor = 0;  // every change of a revision <= floor may be gone
  static constexpr size_t kWatchCap = 1u << 20;
  void log_changes(const std::vector<zg_update>& u, const std::vector<uint8_t>& changed) {
    for (size_t i = 0; i < u.size(); ++i)
      if (changed[i]) watch_log.push_back(WatchEntry{revision, u[i].t, u[i].expires_at, u[i].op});
    while (watch_log.size() > kWatchCap) {
      watch_floor = watch_log.front().revision;
      watch_log.pop_front();
    }
    // a revision is dropped whole: a reader never sees part of a write
    while (!watch_log.empty() && watch_log.front().revision <= watch_floor) watch_log.pop_front();
  }
  // An import: every relationship a CREATE. One larger than the feed holds cannot be read change by change: readers
  // restart from its revision, as after zg_clear_relationships.
  void log_import(const std::vector<zg_tuple>& t, const std::vector<uint32_t>& ex) {
    if (t.size() > kWatchCap) {
      watch_log.clear();
      watch_floor = revision;
      return;
    }
    for (size_t i = 0; i < t.size(); ++i) watch_log.push_back(WatchEntry{revision, t[i], ex[i], ZG_OP_CREATE});
    while (watch_log.size() > kWatchCap) {
      watch_floor = watch_log.front().revision;
      watch_log.pop_front();
    }
    while (!watch_log.empty() && watch_log.front().revision <= watch_floor) watch_log.pop_front();
  }
};

// fn(device, index) on every device of the engine, concurrently; returns when all are done.
static void on_all_devices(zg_engine* e, const std::function<void(Device&, size_t)>& fn) {
  for (size_t i = 0; i < e->replicas.size(); ++i) {
    Replica* r = e->replicas[i].get();
    r->worker.submit([r, i, &fn] { fn(r->dev, i + 1); });
  }
  fn(e->dev, 0);
  for (auto& r : e->replicas) r->worker.wait();
}

#define LOCK_DEVICE(e) std::lock_guard<FairMutex> g((e)->mu)
#define LOCK_NAMES_SHARED(e) std::shared_lock<std::shared_mutex> ng((e)->names)
#define LOCK_NAMES_UNIQUE(e) std::unique_lock<std::shared_mutex> ng((e)->names)

static thread_local std::string g_err;
static constexpr size_t kMaxLookupGroup = 64;  // = kMaxLookupBatch (kernels.cuh)
static const char* kHostOnlyMsg = "host-only engine: no CUDA device, and libzgpu has no CPU fallback";
static const char* kShardedMsg =
    "sharded engine: use zg_shard_route_dev / zg_shard_pass_dev / zg_shard_fold_dev / zg_shard_unroute_dev "
    "(dist.DeviceShardedChecker)";
static const char* kHandleLookupMsg =
    "sharded handle (zg_config.n_shards > 1): LookupResources, LookupSubjects and the list pre-filter are not served "
    "by it; run them on one engine per shard (dist.DeviceShardedLookup) or on a replica";
static const char* kHandleDeviceMsg =
    "sharded handle (zg_config.n_shards > 1): calls on device buffers and the device-ingress calls are not served by "
    "it; use zg_check_bulk, zg_check_bulk_str or zg_check_bulk_packed";
static const char* kHandleShardCallMsg =
    "sharded handle (zg_config.n_shards > 1): the zg_shard_*_dev calls drive one shard per engine; this handle runs "
    "the sharded protocol itself (zg_check_bulk)";
static const char* kHandleSubjectsMsg =
    "sharded handle (zg_config.n_shards > 1): LookupSubjects is not served by it, with or without "
    "ZG_FLAG_HANDLE_LOOKUPS; run it on one engine per shard (dist.DeviceShardedLookup) or on a replica";
static const char* kHandleExpandMsg =
    "sharded handle (zg_config.n_shards > 1): ExpandPermissionTree is not served by it; run it on a replica";
static bool is_handle(const zg_engine* e) { return e->n_shards > 1; }
// a sharded handle that answers LookupSubjects itself (run_sharded_subjects)
static bool serves_subjects(const zg_engine* e) { return is_handle(e) && e->handle_subjects; }
// shard k of a sharded handle
static Device& shard(zg_engine* e, uint32_t k) { return k == 0 ? e->dev : e->replicas[k - 1]->dev; }

static int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

// The kinds of call an engine refuses by its mode: host-only, sharded handle (zg_config.n_shards > 1), or one shard of
// several (zg_config.shard_count > 1).
enum class Call {
  kDevice,         // device work that any device engine serves
  kDeviceBuffers,  // device buffers, no check answered: zg_count_alg_bytes, zg_resolve_checks_packed_device
  kDeviceChecks,   // checks on device buffers or through the device ingress
  kCheckGroup,     // a check group of zg_check_bulk, and the string calls that publish before queueing one
  kLookup,         // LookupResources and the list pre-filter
  kSubjects,       // LookupSubjects
  kExpand,         // ExpandPermissionTree
  kShardCall,      // zg_shard_*_dev: one shard per engine, driven by dist.py
};

// ZG_OK when e serves calls of kind c, else the code it refuses them with; the message goes to *msg when given (the
// callers of a group), else to zg_last_error. A host-only engine is never one shard of several (it has no device).
static int refuse(const zg_engine* e, Call c, std::string* msg = nullptr) {
  const char* why = nullptr;
  if (e->host_only) {
    why = kHostOnlyMsg;
  } else if (is_handle(e)) {
    switch (c) {
      case Call::kDeviceBuffers:
      case Call::kDeviceChecks: why = kHandleDeviceMsg; break;
      case Call::kLookup: why = e->handle_lookups ? nullptr : kHandleLookupMsg; break;
      case Call::kSubjects: why = e->handle_subjects ? nullptr : e->handle_lookups ? kHandleSubjectsMsg : kHandleLookupMsg; break;
      case Call::kShardCall: why = kHandleShardCallMsg; break;
      case Call::kExpand: why = kHandleExpandMsg; break;
      default: break;
    }
  } else if (e->dev.shard_count > 1 && c != Call::kDevice && c != Call::kDeviceBuffers && c != Call::kShardCall) {
    why = kShardedMsg;
  }
  if (!why) return ZG_OK;
  if (msg) *msg = why;
  else g_err = why;
  return e->host_only ? ZG_ECUDA : ZG_EINVAL;
}

// The devices a step runs on: every device of the engine (concurrently), device 0 alone, or shard k >= 0 alone.
constexpr int kEveryDevice = -1, kFirstDevice = -2;

// Runs fn(device, k, &err) -> ZG_* on the devices `which` names (k: the device's index, shard k of a handle). Returns
// the first failing device's code in device order, and that device's message in *err.
template <class F>
static int on_devices(zg_engine* e, int which, F&& fn, std::string* err) {
  if (which != kEveryDevice) {
    const uint32_t k = which == kFirstDevice ? 0 : static_cast<uint32_t>(which);
    std::string m;
    const int rc = fn(shard(e, k), static_cast<size_t>(k), &m);
    if (rc) *err = std::move(m);
    return rc;
  }
  std::vector<int> rcs(1 + e->replicas.size(), ZG_OK);
  std::vector<std::string> errs(rcs.size());
  on_all_devices(e, [&](Device& dev, size_t k) { rcs[k] = fn(dev, k, &errs[k]); });
  for (size_t k = 0; k < rcs.size(); ++k)
    if (rcs[k]) {
      *err = std::move(errs[k]);
      return rcs[k];
    }
  return ZG_OK;
}
extern "C" const char* zg_last_error(void) { return g_err.c_str(); }
extern "C" size_t zg_last_error_copy(char* buf, size_t cap) {
  const size_t n = g_err.size();
  if (buf && cap) {
    const size_t m = n < cap - 1 ? n : cap - 1;
    std::memcpy(buf, g_err.data(), m);
    buf[m] = 0;
  }
  return n;
}

// The string calls resolve names under the shared names lock, release it, and answer later: a check queued for the
// batcher, a lookup whose ids are turned back into names under the lock again. A retirement in between may free a
// resolved name and hand its id to a new name, so the call would answer for, or print, the other name. Runs `call`
// until no retirement happened between its start and its end (a retirement bumps name_epoch before any freed id can
// be reused): then every id it resolved denoted the same name until it answered. A retry redoes the whole call.
template <class F>
static int with_stable_names(zg_engine* e, F&& call) {
  if (!e) return call();
  for (;;) {
    const uint64_t epoch = e->name_epoch.load();
    const int rc = call();
    if (e->name_epoch.load() == epoch) return rc;
  }
}

static uint32_t now_of(const zg_engine* e) {
  return static_cast<uint32_t>(e->clock ? e->clock : static_cast<int64_t>(time(nullptr)));
}
static bool none_rel(const char* s) { return !s || !*s || std::strcmp(s, "...") == 0; }

extern "C" int zg_engine_create(const zg_config* cfg, zg_engine** out) {
  if (!out) return fail(ZG_EINVAL, "out is NULL");
  *out = nullptr;
  const uint32_t S = cfg && cfg->n_shards > 1 ? cfg->n_shards : 1;
  if (S > 1 && cfg->shard_count > 1)
    return fail(ZG_EINVAL, "n_shards > 1 holds every shard in this one handle, shard_count > 1 makes this engine one "
                           "shard of several: set only one of them");
  if (S > static_cast<uint32_t>(kMaxShards)) return fail(ZG_EINVAL, "n_shards exceeds 64 (the routing kernels' destinations)");
  const bool handle_lookups = cfg && (cfg->flags & ZG_FLAG_HANDLE_LOOKUPS);
  if (handle_lookups && S < 2) return fail(ZG_EINVAL, "ZG_FLAG_HANDLE_LOOKUPS needs n_shards > 1");
  const bool handle_subjects = cfg && (cfg->flags & ZG_FLAG_HANDLE_SUBJECTS);
  if (handle_subjects && S < 2) return fail(ZG_EINVAL, "ZG_FLAG_HANDLE_SUBJECTS needs n_shards > 1");
  zg_engine* e = new (std::nothrow) zg_engine();
  if (!e) return fail(ZG_ENOMEM, "out of memory");
  e->n_shards = S;
  e->handle_lookups = handle_lookups;
  e->handle_subjects = handle_subjects;
  if (cfg && (cfg->flags & ZG_FLAG_HOST_ONLY)) {
    e->host_only = true;
    e->keep_built = true;
    *out = e;
    return ZG_OK;
  }
  std::string err = e->dev.init(cfg ? cfg->device : -1, cfg ? cfg->subquery_capacity : 0, cfg ? cfg->work_budget : 0);
  if (!err.empty()) {
    delete e;
    return fail(ZG_ECUDA, err);
  }
  if (cfg && (cfg->flags & ZG_FLAG_FORWARD_ONLY)) e->dev.invert = false;
  if (cfg && cfg->shard_count > 1) {
    if (cfg->shard_rank >= cfg->shard_count) {
      delete e;
      return fail(ZG_EINVAL, "shard_rank must be < shard_count");
    }
    e->dev.shard_count = cfg->shard_count;
    e->dev.shard_rank = cfg->shard_rank;
  }
  if (S > 1) {
    // shard k on device first + k % D; every pair of distinct devices reads and writes the other's memory
    int visible = 0;
    cudaGetDeviceCount(&visible);
    const int first = e->dev.device;
    const int D = cfg->n_devices == ZG_ALL_DEVICES ? visible - first : std::max<int>(1, static_cast<int>(cfg->n_devices));
    if (D < 1 || first + D > visible) {
      delete e;
      return fail(ZG_EINVAL, "n_devices exceeds the visible CUDA devices");
    }
    const int used = std::min<int>(D, static_cast<int>(S));
    for (int a = first; a < first + used; ++a)
      for (int b = first; b < first + used; ++b) {
        if (a == b) continue;
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, a, b) != cudaSuccess || !can) {
          delete e;
          return fail(ZG_EINVAL, "n_shards over several devices: device " + std::to_string(a) + " cannot access the memory of device " +
                                     std::to_string(b) + " (peer access), which the sharded handle's exchange needs");
        }
        cudaSetDevice(a);
        const cudaError_t pe = cudaDeviceEnablePeerAccess(b, 0);  // this process's context only
        if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) {
          delete e;
          return fail(ZG_ECUDA, std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(pe));
        }
        cudaGetLastError();
      }
    cudaSetDevice(first);
    e->shard_devices = static_cast<uint32_t>(used);
    for (uint32_t k = 1; k < S; ++k) {
      e->replicas.emplace_back(new Replica());
      e->replicas.back()->worker.start();
    }
    const zg_config c = *cfg;
    if (on_devices(e, kEveryDevice, [&](Device& dev, size_t k, std::string* m) {
          if (k) *m = dev.init(first + static_cast<int>(k % static_cast<size_t>(D)), c.subquery_capacity, c.work_budget);
          if (c.flags & ZG_FLAG_FORWARD_ONLY) dev.invert = false;
          dev.shard_rank = dev.own_rank = static_cast<uint32_t>(k);
          dev.shard_count = dev.own_count = S;
          return m->empty() ? ZG_OK : ZG_ECUDA;
        }, &err)) {
      delete e;
      return fail(ZG_ECUDA, err);
    }
  } else if (cfg && cfg->n_devices > 1) {
    if (cfg->shard_count > 1) {
      delete e;
      return fail(ZG_EINVAL, "n_devices > 1 makes replicas; a sharded engine owns one device");
    }
    int visible = 0;
    cudaGetDeviceCount(&visible);
    const int first = e->dev.device;
    const int want = cfg->n_devices == ZG_ALL_DEVICES ? visible - first : static_cast<int>(cfg->n_devices);
    if (want < 1 || first + want > visible) {
      delete e;
      return fail(ZG_EINVAL, "n_devices exceeds the visible CUDA devices");
    }
    for (int d = 1; d < want; ++d) {
      e->replicas.emplace_back(new Replica());
      e->replicas.back()->worker.start();
    }
    const zg_config c = *cfg;
    if (on_devices(e, kEveryDevice, [&](Device& dev, size_t i, std::string* m) {
          if (i == 0) return ZG_OK;
          *m = dev.init(first + static_cast<int>(i), c.subquery_capacity, c.work_budget);
          if (c.flags & ZG_FLAG_FORWARD_ONLY) dev.invert = false;
          return m->empty() ? ZG_OK : ZG_ECUDA;
        }, &err)) {
      delete e;
      return fail(ZG_ECUDA, err);
    }
  }
  *out = e;
  return ZG_OK;
}
extern "C" void zg_engine_destroy(zg_engine* e) {
  if (e && std::getenv("ZGPU_BATCHER_STATS"))
    std::fprintf(stderr, "zgpu batcher: %llu groups, %llu callers waited, %llu hand-overs\n",
                 static_cast<unsigned long long>(e->batcher.groups), static_cast<unsigned long long>(e->batcher.waited),
                 static_cast<unsigned long long>(e->batcher.handed_over));
  delete e;
}

extern "C" int zg_load_schema(zg_engine* e, const char* dsl, size_t len) {
  if (!e || !dsl) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  Schema s;
  std::string err = s.parse(std::string(dsl, len));
  if (!err.empty()) return fail(ZG_EINVAL, err);
  e->schema = std::move(s);
  e->has_schema = true;
  ++e->schema_gen;
  e->store.reset(&e->schema);
  e->retire_device = e->retire_host = 0;  // with the store's count of retired names
  ++e->name_epoch;                        // every name is gone
  if (!is_handle(e)) {  // a sharded handle's store holds every shard's relationships
    e->store.shard_count = e->dev.shard_count;
    e->store.shard_rank = e->dev.shard_rank;
  }
  e->dev.snap.reset();
  e->dev.ingress_reset();  // the device mirror of the names
  for (auto& r : e->replicas) r->dev.snap.reset();
  e->shard_built.clear();
  e->dirty = true;
  return ZG_OK;
}

#define NEED_SCHEMA(e, ret)              \
  if (!(e) || !(e)->has_schema) {        \
    g_err = "no schema loaded";          \
    return ret;                          \
  }

extern "C" int zg_num_types(const zg_engine* e) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  return static_cast<int>(e->schema.types.size());
}
extern "C" int zg_num_slots(const zg_engine* e) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  return static_cast<int>(e->schema.slots.size());
}
extern "C" int zg_type_id(const zg_engine* e, const char* n) {
  NEED_SCHEMA(e, -1);
  return n ? e->schema.type_id(n) : -1;
}
extern "C" int zg_slot_id(const zg_engine* e, int t, const char* n) {
  NEED_SCHEMA(e, -1);
  return n ? e->schema.slot_id(t, n) : -1;
}
extern "C" int zg_slot_type(const zg_engine* e, int s) {
  NEED_SCHEMA(e, -1);
  return s >= 0 && s < static_cast<int>(e->schema.slots.size()) ? e->schema.slots[s].type : -1;
}
extern "C" int zg_slot_is_permission(const zg_engine* e, int s) {
  NEED_SCHEMA(e, -1);
  return s >= 0 && s < static_cast<int>(e->schema.slots.size()) ? e->schema.slots[s].is_perm : -1;
}
extern "C" const char* zg_slot_name(const zg_engine* e, int s) {
  NEED_SCHEMA(e, nullptr);
  return s >= 0 && s < static_cast<int>(e->schema.slots.size()) ? e->schema.slots[s].name.c_str() : nullptr;
}
extern "C" const char* zg_type_name(const zg_engine* e, int t) {
  NEED_SCHEMA(e, nullptr);
  return t >= 0 && t < static_cast<int>(e->schema.types.size()) ? e->schema.types[t].name.c_str() : nullptr;
}

extern "C" uint32_t zg_intern_object(zg_engine* e, int t, const char* id) {
  NEED_SCHEMA(e, ZG_NO_OBJECT);
  if (!id || !*id || t < 0 || t >= static_cast<int>(e->schema.types.size())) return ZG_NO_OBJECT;
  LOCK_NAMES_UNIQUE(e);
  return e->store.intern(t, id);
}
extern "C" uint32_t zg_find_object(const zg_engine* e, int t, const char* id) {
  NEED_SCHEMA(e, ZG_NO_OBJECT);
  if (!id) return ZG_NO_OBJECT;
  LOCK_NAMES_SHARED(e);
  return e->store.find(t, id);
}
extern "C" int zg_object_name(const zg_engine* e, int t, uint32_t id, char* buf, size_t cap) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  LOCK_NAMES_SHARED(e);
  std::string_view n;
  if (!e->store.name(t, id, &n)) return fail(ZG_EINVAL, "object has no name");
  if (n.size() + 1 > cap || !buf) return ZG_E2BIG;
  std::memcpy(buf, n.data(), n.size());
  buf[n.size()] = 0;
  return static_cast<int>(n.size());
}

extern "C" int zg_load_tuples(zg_engine* e, const zg_tuple* t, const uint32_t* expires, uint64_t n) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!t && n) return fail(ZG_EINVAL, "NULL tuples");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  std::string err = e->store.load(t, expires, n);
  if (!err.empty()) return fail(ZG_EINVAL, err);
  e->dirty = true;
  return ZG_OK;
}
extern "C" int zg_apply_updates(zg_engine* e, const zg_update* u, uint64_t n) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!u && n) return fail(ZG_EINVAL, "NULL updates");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  int code = ZG_OK;
  std::string err = e->store.apply(u, n, &code);
  if (!err.empty()) return fail(code, err);
  e->dirty = true;
  return ZG_OK;
}

// A sharded handle answers from every shard's snapshot of one revision or from none: after a failed publish no
// shard answers until a publish succeeds.
static int publish_failed(zg_engine* e, const std::string& err) {
  if (is_handle(e))
    for (uint32_t k = 0; k < e->n_shards; ++k) shard(e, k).snap.reset();
  return fail(ZG_ECUDA, err);
}

// Caller holds e->mu AND e->names exclusively.
static int publish_locked(zg_engine* e) {
  (void)e->store.layout();  // settles the object capacities once: the replicas' publishes below only read the store
  if (!e->host_only) {
    // default: build the CSR on the GPU (csrc/build.cu). ZGPU_HOST_BUILD=1 builds on the host
    // and uploads; ZGPU_VERIFY_BUILD=1 does both and compares every array (tests).
    const char* hb = std::getenv("ZGPU_HOST_BUILD");
    const char* vb = std::getenv("ZGPU_VERIFY_BUILD");
    if (!(hb && *hb && *hb != '0')) {
      const bool verify = vb && *vb && *vb != '0';
      // a few updates against a resident snapshot: merge them in (build.cu gpu_apply_delta); anything the
      // journal cannot express (bulk load, new layout, no snapshot yet) rebuilds
      const char* nd = std::getenv("ZGPU_NO_DELTA");
      const bool no_delta = nd && *nd && *nd != '0';
      // every replica merges / builds for itself, concurrently
      std::string err;
      if (on_devices(e, kEveryDevice, [&](Device& dev, size_t, std::string* m) {
            *m = no_delta ? std::string("full") : dev.publish_delta(e->store, e->schema, e->revision + 1);
            if (*m == "full") *m = dev.publish_gpu(e->store, e->schema, e->revision + 1, verify);
            else if (m->empty() && verify) *m = dev.verify_against_host(e->store, e->schema);
            return m->empty() ? ZG_OK : ZG_ECUDA;
          }, &err))
        return publish_failed(e, err);
      ++e->revision;
      e->store.journal_clear();
      e->last_built = HostSnapshot();
      e->shard_built.clear();
      e->dirty = false;
      return ZG_OK;
    }
    if (is_handle(e)) {  // host-built shards: each holds the relationships it owns
      std::string err;
      if (on_devices(e, kEveryDevice, [&](Device& dev, size_t, std::string* m) {
            HostSnapshot h = e->store.build(dev.own_rank, dev.own_count);
            *m = h.err.empty() ? dev.publish(h, e->schema, e->revision + 1) : h.err;
            return m->empty() ? ZG_OK : ZG_ECUDA;
          }, &err))
        return publish_failed(e, err);
      ++e->revision;
      e->store.journal_clear();
      e->shard_built.clear();
      e->dirty = false;
      return ZG_OK;
    }
  }
  e->shard_built.clear();
  HostSnapshot h = e->store.build();
  if (!h.err.empty()) return fail(ZG_EINVAL, h.err);
  if (e->host_only) {
    ++e->revision;
    e->last_built = std::move(h);
    e->dirty = false;
    return ZG_OK;
  }
  std::string err = e->dev.publish(h, e->schema, ++e->revision);
  if (!err.empty()) return fail(ZG_ECUDA, err);
  if (e->keep_built) e->last_built = std::move(h);
  e->dirty = false;
  return ZG_OK;
}
extern "C" int zg_publish(zg_engine* e) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  return publish_locked(e);
}
extern "C" int zg_clear_relationships(zg_engine* e) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  e->store.clear_relationships();
  e->dirty = true;
  // the feed cannot describe "everything went away" change by change: readers restart from here
  e->watch_log.clear();
  int rc = publish_locked(e);
  e->watch_floor = e->revision;
  return rc;
}
extern "C" uint64_t zg_num_tuples(const zg_engine* e) {
  if (!e || !e->has_schema) return 0;
  LOCK_NAMES_UNIQUE(e);  // match() folds the duplicates of bulk loads into the index
  std::vector<uint64_t> idx;
  Store::Filter f;
  e->store.match(f, 0, &idx);  // also folds duplicates of bulk loads
  return e->store.size();
}
extern "C" void zg_set_clock(zg_engine* e, int64_t t) {
  if (e) e->clock = t;
}

// ---- string resolution ---------------------------------------------------------------

static std::string rel_text(const zg_rel_str& r) {
  auto s = [](const char* x) { return std::string(x ? x : ""); };
  return s(r.res_type) + ":" + s(r.res_id) + "#" + s(r.relation) + "@" + s(r.subj_type) + ":" + s(r.subj_id) +
         (none_rel(r.subj_rel) ? "" : "#" + s(r.subj_rel));
}

// SpiceDB object-id validation (v1 API): 1..1024 characters of [a-zA-Z0-9/_|\-=+], or "*".
static bool valid_object_id(const char* id, size_t n) {
  if (n == 0 || n > 1024) return false;
  if (n == 1 && id[0] == '*') return true;
  for (size_t i = 0; i < n; ++i) {
    const unsigned char c = static_cast<unsigned char>(id[i]);
    if (!(std::isalnum(c) || c == '/' || c == '_' || c == '|' || c == '-' || c == '=' || c == '+')) return false;
  }
  return true;
}
static bool valid_object_id(const char* id) { return valid_object_id(id, std::strlen(id)); }

// Resolve a relationship to WRITE (interns objects). Returns "" or an error.
static std::string resolve_write(zg_engine* e, const zg_rel_str& r, zg_tuple* t) {
  const Schema& sc = e->schema;
  if (!r.res_type || !r.res_id || !r.relation || !r.subj_type || !r.subj_id) return "relationship has NULL fields";
  int rt = sc.type_id(r.res_type), st = sc.type_id(r.subj_type);
  if (rt < 0) return std::string("object definition `") + r.res_type + "` not found";
  if (st < 0) return std::string("object definition `") + r.subj_type + "` not found";
  int rel = sc.slot_id(rt, r.relation);
  if (rel < 0 || sc.slots[rel].is_perm)
    return std::string("relation `") + r.relation + "` not found under definition `" + r.res_type + "`";
  if (!valid_object_id(r.res_id) || std::strcmp(r.res_id, "*") == 0)
    return std::string("invalid resource object id `") + r.res_id + "`";
  if (!valid_object_id(r.subj_id)) return std::string("invalid subject object id `") + r.subj_id + "`";
  t->rel = static_cast<uint16_t>(rel);
  t->stype = static_cast<uint16_t>(st);
  t->flags = 0;
  t->srel = kNone;
  if (std::strcmp(r.subj_id, "*") == 0) {
    if (!none_rel(r.subj_rel)) return "wildcard subjects cannot have a relation";
    t->srel = kWildcard;
    t->subj = 0;
  } else {
    if (!none_rel(r.subj_rel)) {
      int sr = sc.slot_id(st, r.subj_rel);
      if (sr < 0) return std::string("relation `") + r.subj_rel + "` not found under definition `" + r.subj_type + "`";
      t->srel = static_cast<uint16_t>(sr);
    }
    t->subj = e->store.intern(st, r.subj_id);
  }
  t->res = e->store.intern(rt, r.res_id);
  return "";
}

// SpiceDB's pattern for optional_resource_id_prefix: 1..1024 characters of [a-zA-Z0-9/_|\-=+] ("*" is not one).
static bool valid_id_prefix(const char* p) {
  const size_t n = std::strlen(p);
  return n <= 1024 && valid_object_id(p, n) && std::strcmp(p, "*") != 0;
}

static Store::Filter resolve_filter(const zg_engine* e, const zg_filter_ex& fx, std::string* err) {
  const Schema& sc = e->schema;
  const zg_filter_str& f = fx.f;
  Store::Filter o;
  auto set = [](const char* s) { return s && *s; };
  if (set(fx.res_id_prefix)) {
    if (!valid_id_prefix(fx.res_id_prefix)) {
      *err = std::string("invalid resource id prefix `") + fx.res_id_prefix + "`";
      return o;
    }
    if (set(f.res_id)) {
      *err = "resource id and resource id prefix cannot both be given";
      return o;
    }
    o.prefix = fx.res_id_prefix;
  }
  if (set(f.res_type)) {
    o.res_type = sc.type_id(f.res_type);
    if (o.res_type < 0) {
      *err = std::string("object definition `") + f.res_type + "` not found";
      return o;
    }
  }
  if (set(f.res_id)) {
    if (o.res_type < 0) {
      *err = "resource id filter needs a resource type";
      return o;
    }
    o.has_res = true;
    o.res = e->store.find(o.res_type, f.res_id);
    if (o.res == ZG_NO_OBJECT) o.impossible = true;
  }
  if (set(f.relation)) {
    if (o.res_type < 0) {
      *err = "relation filter needs a resource type";
      return o;
    }
    o.rel = sc.slot_id(o.res_type, f.relation);
    if (o.rel < 0) {
      *err = std::string("relation `") + f.relation + "` not found under definition `" + f.res_type + "`";
      return o;
    }
  }
  if (set(f.subj_type)) {
    o.subj_type = sc.type_id(f.subj_type);
    if (o.subj_type < 0) {
      *err = std::string("object definition `") + f.subj_type + "` not found";
      return o;
    }
  }
  if (set(f.subj_id)) {
    if (o.subj_type < 0) {
      *err = "subject id filter needs a subject type";
      return o;
    }
    if (std::strcmp(f.subj_id, "*") == 0) {
      o.subj_wildcard = true;
    } else {
      o.has_subj = true;
      o.subj = e->store.find(o.subj_type, f.subj_id);
      if (o.subj == ZG_NO_OBJECT) o.impossible = true;
    }
  }
  if (set(f.subj_rel)) {
    if (o.subj_type < 0) {
      *err = "subject relation filter needs a subject type";
      return o;
    }
    o.has_srel = true;
    if (std::strcmp(f.subj_rel, "...") == 0) {
      o.srel = kNone;
    } else {
      int sr = sc.slot_id(o.subj_type, f.subj_rel);
      if (sr < 0) o.impossible = true;
      else o.srel = static_cast<uint16_t>(sr);
    }
  }
  return o;
}

// A relationship filter is answered from the snapshot on the device when that snapshot is the store: the engine has a
// device, every shard holds the snapshot of the current revision, and nothing was loaded or applied since it was
// published. Otherwise Store::match answers: host-only engines, and stores with unpublished changes (a read never
// publishes: relationships loaded and not yet published stay invisible to checks). Caller holds e->mu.
static bool filters_on_device(const zg_engine* e) {
  if (e->host_only || e->dirty.load()) return false;
  const uint32_t n = is_handle(e) ? e->n_shards : 1;
  for (uint32_t k = 0; k < n; ++k) {
    const auto& s = shard(const_cast<zg_engine*>(e), k).snap;
    if (!s || s->revision != e->revision) return false;
  }
  return true;
}

// A device's part of a filter or a collection: Device::match_filter or Device::match_expired.
using DeviceMatch = std::function<int(Device&, uint64_t* count, std::vector<zg_tuple>* tuples, bool* too_big, std::string* err)>;

// The devices that answer from the resident snapshot (on_devices): replicas hold the same snapshot, so the first
// device answers; every shard of a sharded handle holds its own relationships, and when the filter `f` names the
// resource, its owner alone.
static int snapshot_devices(const zg_engine* e, const Store::Filter* f = nullptr) {
  if (!is_handle(e)) return kFirstDevice;
  return f && f->has_res ? static_cast<int>(f->res % e->n_shards) : kEveryDevice;
}

// Runs `ask` on the snapshot devices `which`, adds up the counts and concatenates the records, and counts a device
// filter of `shape`.
static int ask_devices(zg_engine* e, int which, Device::FilterShape shape, const DeviceMatch& ask, uint64_t* count,
                       std::vector<zg_tuple>* tuples, bool* too_big) {
  *count = 0;
  *too_big = false;
  if (tuples) tuples->clear();
  const uint32_t S = is_handle(e) ? e->n_shards : 1;
  std::vector<uint64_t> n(S, 0);
  std::vector<std::vector<zg_tuple>> got(tuples ? S : 0);
  std::vector<char> big(S, 0);
  std::string err;
  if (int rc = on_devices(e, which, [&](Device& dev, size_t k, std::string* m) {
        bool b = false;
        const int arc = ask(dev, &n[k], tuples ? &got[k] : nullptr, &b, m);
        big[k] = b;
        return arc;
      }, &err))
    return fail(rc == ZG_ENOMEM ? ZG_ECUDA : rc, err);
  for (uint32_t k = 0; k < S; ++k) {
    *count += n[k];
    *too_big = *too_big || big[k];
  }
  if (*too_big) return ZG_OK;
  ++e->flt_device;
  ++e->flt_shape[shape];
  if (tuples) {
    for (auto& g : got) tuples->insert(tuples->end(), g.begin(), g.end());
    e->flt_returned += tuples->size();
  }
  return ZG_OK;
}

// A filter answered by the host store: counted in zg_filter_counters, and in zg_prefix_counters with a prefix.
static void count_host(zg_engine* e, const Store::Filter& f) {
  ++e->flt_host;
  if (!f.prefix.empty()) ++e->px_host;
}

// The bitmaps of f's prefix (Device::prefix_scan), built once on the first device from the handle's names; every shard
// of a sharded handle reads them there through peer memory (replicas answer on that device). *too_big: over the
// output budget, and the caller answers on the host. Caller holds e->mu and e->names (shared is enough).
static int prefix_on_device(zg_engine* e, const Store::Filter& f, PrefixBits* px, bool* too_big) {
  PrefixStats st;
  std::string err;
  const int rc = e->dev.prefix_scan(e->store, e->schema, f.res_type, f.prefix, px, &st, too_big, &err);
  e->px_names += st.names;
  e->px_matched += st.matched;
  e->px_launches += st.launches;
  e->px_syncs += st.syncs;
  return rc ? fail(rc == ZG_ENOMEM ? ZG_ECUDA : rc, err) : ZG_OK;
}

// The device path of a filter. Caller holds e->mu and e->names (shared is enough) and has seen filters_on_device.
// *count = the matching relationships; with `tuples`, the records in no particular order. A sharded handle asks every
// shard (they own disjoint relationships), or the owner alone when the resource is given; replicas hold the same
// snapshot, so the first device answers. *too_big: the records would not fit the device's output budget and the
// caller runs Store::match instead (holding e->names exclusively).
static int match_on_device(zg_engine* e, const Store::Filter& f, uint32_t now, uint64_t* count, std::vector<zg_tuple>* tuples,
                           bool* too_big) {
  PrefixBits px;
  const bool has_prefix = !f.prefix.empty();
  if (has_prefix) {
    *count = 0;
    if (int rc = prefix_on_device(e, f, &px, too_big)) return rc;
    if (*too_big) return ZG_OK;
  }
  const int rc = ask_devices(e, snapshot_devices(e, &f), Device::filter_shape(f), [&](Device& dev, uint64_t* n, std::vector<zg_tuple>* got, bool* big,
                                                            std::string* err) {
    return dev.match_filter(e->schema, f, now, n, got, nullptr, big, err, has_prefix ? &px : nullptr);
  }, count, tuples, too_big);
  if (!rc && has_prefix && !*too_big) ++e->px_device;
  return rc;
}

// Removes the relationships a delete by filter or a collection found. On the device path the records `found` (any
// order) become store positions through the index apply() needs anyway, and in ascending order the updates and the
// watch feed are those of the host scan, which leaves its positions in *idx (found == nullptr). Applies the DELETEs
// (*u, and *changed for the feed), sets *n_done, and publishes once. Caller holds e->mu AND e->names exclusively.
static int delete_found(zg_engine* e, const char* what, const std::vector<zg_tuple>* found, std::vector<uint64_t>* idx,
                        std::vector<zg_update>* u, std::vector<uint8_t>* changed, uint64_t* n_done) {
  if (found && !e->store.locate(found->data(), found->size(), idx))
    return fail(ZG_ECUDA, std::string(what) + ": the snapshot holds a relationship the store does not");
  u->resize(idx->size());
  for (size_t i = 0; i < idx->size(); ++i) {
    (*u)[i].t = e->store.tuples[(*idx)[i]];
    (*u)[i].expires_at = 0;
    (*u)[i].op = ZG_OP_DELETE;
  }
  int code = ZG_OK;
  std::string err = e->store.apply(u->data(), u->size(), &code, changed);
  if (!err.empty()) return fail(code, err);
  e->dirty = true;
  if (n_done) *n_done = idx->size();
  return publish_locked(e);
}

// Caller holds e->mu AND e->names exclusively (every writer does).
static int check_preconditions(zg_engine* e, const zg_precondition_ex* pre, uint64_t n_pre) {
  std::vector<uint64_t> idx;
  const bool on_device = n_pre && filters_on_device(e);
  for (uint64_t i = 0; i < n_pre; ++i) {
    std::string err;
    Store::Filter f = resolve_filter(e, pre[i].filter, &err);
    if (!err.empty()) return fail(ZG_EINVAL, "precondition " + std::to_string(i) + ": " + err);
    uint64_t count = 0;
    bool too_big = false;  // a count needs no output: only a prefix's bitmaps can be over the budget
    if (on_device) {
      if (int rc = match_on_device(e, f, now_of(e), &count, nullptr, &too_big)) return rc;
    }
    if (!on_device || too_big) {
      e->store.match(f, now_of(e), &idx);
      count_host(e, f);
      count = idx.size();
    }
    const bool any = count != 0;
    if (pre[i].op == ZG_PRECOND_MUST_MATCH && !any)
      return fail(ZG_EPRECOND, "precondition " + std::to_string(i) + " (MUST_MATCH) failed");
    if (pre[i].op == ZG_PRECOND_MUST_NOT_MATCH && any)
      return fail(ZG_EPRECOND, "precondition " + std::to_string(i) + " (MUST_NOT_MATCH) failed");
    if (pre[i].op != ZG_PRECOND_MUST_MATCH && pre[i].op != ZG_PRECOND_MUST_NOT_MATCH)
      return fail(ZG_EINVAL, "unknown precondition operation");
  }
  return ZG_OK;
}

// The preconditions of the calls without _ex, with the prefix unset.
static std::vector<zg_precondition_ex> pre_ex(const zg_precondition_str* pre, uint64_t n_pre) {
  std::vector<zg_precondition_ex> x(pre ? n_pre : 0);
  for (size_t i = 0; i < x.size(); ++i) x[i] = zg_precondition_ex{pre[i].op, zg_filter_ex{pre[i].filter, nullptr}};
  return x;
}

extern "C" int zg_write_relationships(zg_engine* e, const zg_update_str* ups, uint64_t n, const zg_precondition_str* pre,
                                      uint64_t n_pre) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!pre && n_pre) return fail(ZG_EINVAL, "NULL argument");
  return zg_write_relationships_ex(e, ups, n, pre_ex(pre, n_pre).data(), n_pre);
}

extern "C" int zg_write_relationships_ex(zg_engine* e, const zg_update_str* ups, uint64_t n, const zg_precondition_ex* pre,
                                         uint64_t n_pre) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if ((!ups && n) || (!pre && n_pre)) return fail(ZG_EINVAL, "NULL argument");
  if (n > 1000)  // pkg/spicedb/spicedb.go:34 WithMaximumUpdatesPerWrite(1000)
    return fail(ZG_EINVAL, "update count of " + std::to_string(n) + " is greater than maximum allowed of 1000");
  if (n_pre > 1000)  // pkg/spicedb/spicedb.go:35
    return fail(ZG_EINVAL, "precondition count is greater than maximum allowed of 1000");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  std::vector<zg_update> u(n);
  for (uint64_t i = 0; i < n; ++i) {
    if (ups[i].op == ZG_OP_DELETE) {
      // deleting a relationship whose objects were never written is a no-op, not an error
      const zg_rel_str& r = ups[i].rel;
      const Schema& sc = e->schema;
      int rt = r.res_type ? sc.type_id(r.res_type) : -1, st = r.subj_type ? sc.type_id(r.subj_type) : -1;
      int rel = rt >= 0 && r.relation ? sc.slot_id(rt, r.relation) : -1;
      if (rt < 0 || st < 0 || rel < 0 || sc.slots[rel].is_perm || !r.res_id || !r.subj_id)
        return fail(ZG_EINVAL, "update " + std::to_string(i) + ": malformed relationship " + rel_text(r));
    }
    std::string err = resolve_write(e, ups[i].rel, &u[i].t);
    if (!err.empty()) return fail(ZG_EINVAL, "update " + std::to_string(i) + " (" + rel_text(ups[i].rel) + "): " + err);
    u[i].expires_at = ups[i].expires_at;
    u[i].op = ups[i].op;
    // two updates of one relationship in a single write are rejected by SpiceDB
    for (uint64_t j = 0; j < i; ++j)
      if (key_of(u[j].t) == key_of(u[i].t))
        return fail(ZG_EINVAL, "found more than one update with relationship " + rel_text(ups[i].rel));
  }
  int rc = check_preconditions(e, pre, n_pre);
  if (rc) return rc;
  int code = ZG_OK;
  std::vector<uint8_t> changed;
  std::string err = e->store.apply(u.data(), n, &code, &changed);
  if (!err.empty()) return fail(code, err);
  e->dirty = true;  // until the publish succeeds the snapshot is not the store: filters_on_device
  rc = publish_locked(e);
  if (rc == ZG_OK) e->log_changes(u, changed);
  return rc;
}

// ---- ImportBulkRelationships ------------------------------------------------------------------------

static constexpr uint64_t kMaxImport = 1ull << 30;  // relationships in one call

// One group's literal fields, resolved once, and what the write path would say of its items by their kind (wildcard
// subject or not, expiring or not).
struct ImportLit {
  int rt = -1, st = -1, rel = -1;
  uint16_t srel = kNone;        // of a non-wildcard subject
  bool has_srel = false;        // the group names a subject relation
  std::string lit_err;          // every item fails with it before its ids are looked at
  std::string srel_err;         // the subject relation does not exist: every non-wildcard item fails with it
  std::string val_err[2][2];    // Store::validate of an item [wildcard][expiring]
  bool all_ok = false;          // no item kind fails: only the ids can
};

static ImportLit import_literals(const zg_engine* e, const zg_import_group& g) {
  const Schema& sc = e->schema;
  ImportLit l;
  if (!g.res_type || !g.relation || !g.subj_type) {
    l.lit_err = "relationship has NULL fields";
    return l;
  }
  l.rt = sc.type_id(g.res_type);
  l.st = sc.type_id(g.subj_type);
  if (l.rt < 0) l.lit_err = std::string("object definition `") + g.res_type + "` not found";
  else if (l.st < 0) l.lit_err = std::string("object definition `") + g.subj_type + "` not found";
  if (!l.lit_err.empty()) return l;
  l.rel = sc.slot_id(l.rt, g.relation);
  if (l.rel < 0 || sc.slots[l.rel].is_perm) {
    l.lit_err = std::string("relation `") + g.relation + "` not found under definition `" + g.res_type + "`";
    return l;
  }
  l.has_srel = !none_rel(g.subj_rel);
  if (l.has_srel) {
    const int sr = sc.slot_id(l.st, g.subj_rel);
    if (sr < 0) l.srel_err = std::string("relation `") + g.subj_rel + "` not found under definition `" + g.subj_type + "`";
    else l.srel = static_cast<uint16_t>(sr);
  }
  l.all_ok = true;
  for (int w = 0; w < 2; ++w)
    for (int x = 0; x < 2; ++x) {
      zg_tuple t{};
      t.rel = static_cast<uint16_t>(l.rel);
      t.stype = static_cast<uint16_t>(l.st);
      t.srel = w ? kWildcard : l.srel;
      if (w ? l.has_srel : !l.srel_err.empty()) {
        l.all_ok = false;
        continue;
      }
      l.val_err[w][x] = e->store.validate(t, x != 0);
      if (!l.val_err[w][x].empty()) l.all_ok = false;
    }
  return l;
}

static bool import_wild(const zg_import_group& g, uint64_t j) {
  return g.subj_off[j + 1] - g.subj_off[j] == 1 && g.subj_ids[g.subj_off[j]] == '*';
}

// What the write path says of item j of group g at call position i, short of the duplicate checks: ZG_OK, or the code
// with the message in *msg. syntax: check the ids too (the device path checks them on the device).
static int import_item_error(const zg_import_group& g, const ImportLit& l, uint64_t j, uint64_t i, bool syntax,
                             std::string* msg) {
  const char* rid = g.res_ids + g.res_off[j];
  const char* sid = g.subj_ids + g.subj_off[j];
  const size_t rl = g.res_off[j + 1] - g.res_off[j], sl = g.subj_off[j + 1] - g.subj_off[j];
  const bool wild = import_wild(g, j), expiring = g.expires_at && g.expires_at[j];
  auto text = [&] {
    const std::string r(rid, rl), su(sid, sl);
    zg_rel_str x{g.res_type, r.c_str(), g.relation, g.subj_type, su.c_str(), g.subj_rel};
    return rel_text(x);
  };
  std::string err = l.lit_err;
  if (err.empty() && syntax) {
    if (!valid_object_id(rid, rl) || (rl == 1 && rid[0] == '*'))
      err = "invalid resource object id `" + std::string(rid, rl) + "`";
    else if (!valid_object_id(sid, sl))
      err = "invalid subject object id `" + std::string(sid, sl) + "`";
  }
  if (err.empty() && wild && l.has_srel) err = "wildcard subjects cannot have a relation";
  if (err.empty() && !wild) err = l.srel_err;
  if (!err.empty()) {
    *msg = "relationship " + std::to_string(i) + " (" + text() + "): " + err;
    return ZG_EINVAL;
  }
  const std::string& v = l.val_err[wild][expiring];
  if (!v.empty()) {
    *msg = "relationship " + std::to_string(i) + ": " + v;
    return ZG_EINVAL;
  }
  return ZG_OK;
}

static int import_exists(uint64_t i) {
  return fail(ZG_EEXIST, "relationship " + std::to_string(i) + ": relationship already exists");
}

// The error of the first failing relationship, at call position `first` (known to fail).
static int import_fail_at(const zg_import_group* g, const std::vector<ImportLit>& lits, const std::vector<uint64_t>& item0,
                          uint64_t first) {
  const size_t k = static_cast<size_t>(std::upper_bound(item0.begin(), item0.end(), first) - item0.begin() - 1);
  std::string msg;
  const int rc = import_item_error(g[k], lits[k], first - item0[k], first, true, &msg);
  return rc ? fail(rc, msg) : import_exists(first);
}

static double ms_since(const std::chrono::steady_clock::time_point& t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// The host path: every relationship in call order through the write path's checks, new names in a per-call table with
// temporary ids above each type's extent, duplicates against the relationship index and within the call. Then the new
// names are interned in first-appearance order, which hands out the ids the write path would. Fills *t (ids final) and
// *new_names; changes nothing else.
static int import_on_host(zg_engine* e, const zg_import_group* g, uint64_t ng, const std::vector<ImportLit>& lits,
                          std::vector<zg_tuple>* t, uint64_t* found, uint64_t* new_names) {
  Store& st = e->store;
  const size_t nt = e->schema.types.size();
  std::vector<uint32_t> extent(nt);
  for (size_t ty = 0; ty < nt; ++ty) extent[ty] = st.extent(static_cast<int>(ty));
  std::vector<std::unordered_map<std::string_view, uint32_t>> fresh(nt);
  std::vector<std::vector<std::string_view>> order(nt);
  auto id_of = [&](int ty, const char* s, size_t len, bool* known) {
    const uint32_t have = st.find(ty, s, len);
    if (have != ZG_NO_OBJECT) {
      ++*found;
      return have;
    }
    *known = false;
    const std::string_view v(s, len);
    auto it = fresh[ty].find(v);
    if (it != fresh[ty].end()) return it->second;
    const uint32_t tmp = extent[ty] + static_cast<uint32_t>(order[ty].size());
    order[ty].push_back(v);
    fresh[ty].emplace(v, tmp);
    return tmp;
  };
  std::unordered_set<Key, KeyHash> seen;
  uint64_t i = 0;
  for (uint64_t k = 0; k < ng; ++k)
    for (uint64_t j = 0; j < g[k].n; ++j, ++i) {
      const ImportLit& l = lits[k];
      std::string msg;
      if (int rc = import_item_error(g[k], l, j, i, true, &msg)) return fail(rc, msg);
      zg_tuple x{};
      x.rel = static_cast<uint16_t>(l.rel);
      x.stype = static_cast<uint16_t>(l.st);
      bool known = true;
      if (import_wild(g[k], j)) {
        x.srel = kWildcard;
      } else {
        x.srel = l.srel;
        x.subj = id_of(l.st, g[k].subj_ids + g[k].subj_off[j], g[k].subj_off[j + 1] - g[k].subj_off[j], &known);
      }
      x.res = id_of(l.rt, g[k].res_ids + g[k].res_off[j], g[k].res_off[j + 1] - g[k].res_off[j], &known);
      if ((known && st.contains(x)) || !seen.insert(key_of(x)).second) return import_exists(i);
      t->push_back(x);
    }
  std::vector<std::vector<uint32_t>> ids(nt);
  for (size_t ty = 0; ty < nt; ++ty) {
    for (std::string_view v : order[ty]) ids[ty].push_back(st.intern(static_cast<int>(ty), std::string(v)));
    *new_names += order[ty].size();
  }
  for (zg_tuple& x : *t) {
    const uint32_t rt = e->schema.slots[x.rel].type;
    if (x.res >= extent[rt]) x.res = ids[rt][x.res - extent[rt]];
    if (x.srel != kWildcard && x.subj >= extent[x.stype]) x.subj = ids[x.stype][x.subj - extent[x.stype]];
  }
  return ZG_OK;
}

// The device path (import.cuh): names, sort and duplicates on the GPU; the host checks the item kinds the literal
// fields decide (no id bytes read but a subject's first) and interns the new names the device found, with their
// hashes, in first-appearance order. Fills *t and the counts; changes nothing but the name mirror's sync on failure.
static int import_on_device(zg_engine* e, const zg_import_group* g, uint64_t ng, const std::vector<ImportLit>& lits,
                            const std::vector<uint64_t>& item0, uint64_t total, bool locate, std::vector<zg_tuple>* t,
                            uint64_t* found, uint64_t* new_names, double* ms) {
  Store& st = e->store;
  const Schema& sc = e->schema;
  // the first item the literal fields fail: only the items before it can be the first to fail
  uint64_t first = total;
  for (uint64_t k = 0; k < ng && first == total; ++k) {
    const ImportLit& l = lits[k];
    if (l.all_ok || !g[k].n) continue;
    if (!l.lit_err.empty()) {
      first = item0[k];
      break;
    }
    for (uint64_t j = 0; j < g[k].n; ++j) {
      const bool wild = import_wild(g[k], j), expiring = g[k].expires_at && g[k].expires_at[j];
      if ((wild ? l.has_srel : !l.srel_err.empty()) || !l.val_err[wild][expiring].empty()) {
        first = item0[k] + j;
        break;
      }
    }
  }
  std::vector<Device::ImportGroup> dg;
  for (uint64_t k = 0; k < ng && item0[k] < first; ++k) {
    if (!g[k].n) continue;
    const ImportLit& l = lits[k];
    Device::ImportGroup d{};
    d.res_ids = g[k].res_ids;
    d.subj_ids = g[k].subj_ids;
    d.res_off = g[k].res_off;
    d.subj_off = g[k].subj_off;
    d.item0 = item0[k];
    d.n = std::min<uint64_t>(g[k].n, first - item0[k]);
    d.rtype = static_cast<uint32_t>(l.rt);
    d.stype = static_cast<uint32_t>(l.st);
    d.rel = static_cast<uint32_t>(l.rel);
    d.rel_index = static_cast<uint32_t>(sc.slots[l.rel].rel_index);
    d.srel = l.srel;
    d.pos_plain = static_cast<uint32_t>(page_class_pos(sc, l.rel, static_cast<uint16_t>(l.st), l.srel));
    d.pos_wild = static_cast<uint32_t>(page_class_pos(sc, l.rel, static_cast<uint16_t>(l.st), kWildcard));
    d.k_plain = static_cast<uint32_t>(sc.class_of(l.rel, static_cast<uint16_t>(l.st), l.srel));
    d.k_wild = static_cast<uint32_t>(sc.class_of(l.rel, static_cast<uint16_t>(l.st), kWildcard));
    dg.push_back(d);
  }
  const uint64_t n = first;
  const size_t nt = sc.types.size();
  std::vector<uint32_t> extent(nt);
  for (size_t ty = 0; ty < nt; ++ty) extent[ty] = st.extent(static_cast<int>(ty));
  Device::ImportCheck chk;
  std::string err;
  if (int rc = e->dev.import_check(st, dg, n, extent, locate && !is_handle(e), &chk, &err)) return fail(rc == ZG_ENOMEM ? ZG_ECUDA : rc, err);
  uint64_t dup = chk.dup;
  if (locate && is_handle(e)) {
    std::vector<uint64_t> d(e->n_shards, ~0ull);
    if (int rc = on_devices(e, kEveryDevice, [&](Device& dev, size_t k, std::string* m) { return dev.import_locate(e->dev, &d[k], m); }, &err))
      return fail(rc == ZG_ENOMEM ? ZG_ECUDA : rc, err);
    for (uint64_t x : d) dup = std::min(dup, x);
  }
  ms[0] = chk.ms_names;
  ms[1] = chk.ms_sort;
  ms[2] = chk.ms_dups;
  first = std::min({first, chk.bad, dup});
  if (first < total) return import_fail_at(g, lits, item0, first);

  // every check passed: the ids the host hands out, lowest free first, then the extent
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<uint32_t> ids;
  std::vector<uint64_t> base(nt, 0);
  std::vector<uint32_t> next;
  for (size_t ty = 0; ty < nt; ++ty) {
    base[ty] = ids.size();
    st.next_ids(static_cast<int>(ty), chk.type_count[ty], &next);
    ids.insert(ids.end(), next.begin(), next.end());
  }
  std::vector<uint32_t> rtype_of_rel(sc.slots.size());
  for (size_t r = 0; r < sc.slots.size(); ++r) rtype_of_rel[r] = sc.slots[r].type;
  if (int rc = e->dev.import_finish(ids, base, rtype_of_rel, t, &err)) return fail(rc == ZG_ENOMEM ? ZG_ECUDA : rc, err);
  for (size_t j = 0; j < chk.new_keys.size(); ++j) {
    const int ty = static_cast<int>(chk.new_keys[j] >> 48);
    const uint64_t o = chk.new_keys[j] & ((1ull << 48) - 1), item = o >> 1;
    const size_t k = static_cast<size_t>(std::upper_bound(item0.begin(), item0.end(), item) - item0.begin() - 1);
    const uint64_t at = item - item0[k];
    const char* s = (o & 1) ? g[k].res_ids + g[k].res_off[at] : g[k].subj_ids + g[k].subj_off[at];
    const uint32_t len = (o & 1) ? g[k].res_off[at + 1] - g[k].res_off[at] : g[k].subj_off[at + 1] - g[k].subj_off[at];
    st.intern_new(ty, s, len, chk.new_hash[j]);
  }
  *found += chk.found;
  *new_names += chk.new_keys.size();
  ms[3] = ms_since(t0);
  return ZG_OK;
}

extern "C" int zg_import_relationships(zg_engine* e, const zg_import_group* groups, uint64_t n_groups, uint64_t* n_imported) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (n_imported) *n_imported = 0;
  if (!groups && n_groups) return fail(ZG_EINVAL, "NULL groups");
  std::vector<uint64_t> item0(n_groups);
  uint64_t total = 0;
  for (uint64_t k = 0; k < n_groups; ++k) {
    item0[k] = total;
    if (!groups[k].n) continue;
    if (!groups[k].res_ids || !groups[k].res_off || !groups[k].subj_ids || !groups[k].subj_off)
      return fail(ZG_EINVAL, "group " + std::to_string(k) + ": NULL ids or offsets");
    for (uint64_t j = 0; j < groups[k].n; ++j)
      if (groups[k].res_off[j + 1] < groups[k].res_off[j] || groups[k].subj_off[j + 1] < groups[k].subj_off[j])
        return fail(ZG_EINVAL, "group " + std::to_string(k) + ": offsets must not decrease");
    total += groups[k].n;
  }
  // the device path indexes the new-name table (>= 4 slots per relationship) with 32-bit slot numbers
  if (total > kMaxImport) return fail(ZG_EINVAL, "more than 2^30 relationships in one import");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  if (e->store.shard_count > 1)
    return fail(ZG_EINVAL, "import relationships: this engine is one shard of several (zg_config.shard_count) and its store "
                           "does not hold the other shards' relationships");
  std::vector<ImportLit> lits(n_groups);
  for (uint64_t k = 0; k < n_groups; ++k) lits[k] = import_literals(e, groups[k]);
  const char* ih = std::getenv("ZGPU_IMPORT_HOST");
  // the device finds duplicates against the resident snapshot: it must be the store, or the store must be empty
  const bool current = filters_on_device(e);
  const bool on_device = !e->host_only && !(ih && *ih && *ih != '0') && (current || e->store.tuples.empty());
  std::vector<zg_tuple> t;
  t.reserve(total);
  uint64_t found = 0, fresh = 0;
  double ms[7] = {};  // zg_import_last_times: kept only when the import succeeds
  const auto t0 = std::chrono::steady_clock::now();
  struct Release {  // the scratch goes with the call, whatever its outcome
    zg_engine* e;
    ~Release() {
      e->dev.import_release();
      for (auto& r : e->replicas) r->dev.import_release();
    }
  } release{e};
  const int rc = on_device ? import_on_device(e, groups, n_groups, lits, item0, total, current && !e->store.tuples.empty(), &t, &found, &fresh, ms)
                           : import_on_host(e, groups, n_groups, lits, &t, &found, &fresh);
  if (rc) return rc;
  if (!on_device) ms[3] = ms_since(t0);
  std::vector<uint32_t> ex(total, 0);
  for (uint64_t k = 0; k < n_groups; ++k)
    if (groups[k].expires_at) std::memcpy(ex.data() + item0[k], groups[k].expires_at, groups[k].n * 4);
  const auto t1 = std::chrono::steady_clock::now();
  e->store.import(t.data(), ex.data(), total);
  ms[4] = ms_since(t1);
  e->dirty = true;  // until the publish succeeds the snapshot is not the store: filters_on_device
  const auto t2 = std::chrono::steady_clock::now();
  const int prc = publish_locked(e);
  ms[5] = ms_since(t2);
  ms[6] = ms_since(t0);
  if (prc) return prc;
  std::memcpy(e->imp_ms, ms, sizeof(ms));
  e->log_import(t, ex);
  ++(on_device ? e->imp_device : e->imp_host);
  e->imp_rels += total;
  e->imp_found += found;
  e->imp_new += fresh;
  if (n_imported) *n_imported = total;
  return ZG_OK;
}

extern "C" int zg_import_counters(zg_engine* e, uint64_t* out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!out) return fail(ZG_EINVAL, "out is NULL");
  LOCK_DEVICE(e);
  out[0] = e->imp_device;
  out[1] = e->imp_host;
  out[2] = e->imp_rels;
  out[3] = e->imp_found;
  out[4] = e->imp_new;
  return ZG_OK;
}

extern "C" int zg_import_last_times(zg_engine* e, double* ms) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!ms) return fail(ZG_EINVAL, "ms is NULL");
  LOCK_DEVICE(e);
  std::memcpy(ms, e->imp_ms, sizeof(e->imp_ms));
  return ZG_OK;
}

static int delete_all(zg_engine* e, const zg_filter_ex* filter, const zg_precondition_ex* pre, uint64_t n_pre,
                      uint64_t* n_deleted) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!filter || (!pre && n_pre)) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  std::string err;
  Store::Filter f = resolve_filter(e, *filter, &err);
  if (!err.empty()) return fail(ZG_EINVAL, err);
  int rc = check_preconditions(e, pre, n_pre);
  if (rc) return rc;
  std::vector<uint64_t> idx;  // expired relationships are deleted too: clock 0
  std::vector<zg_tuple> found;
  bool on_device = filters_on_device(e);
  if (on_device) {
    uint64_t count = 0;
    bool too_big = false;
    rc = match_on_device(e, f, 0, &count, &found, &too_big);
    if (rc) return rc;
    on_device = !too_big;
  }
  if (!on_device) {
    e->store.match(f, 0, &idx);
    count_host(e, f);
  }
  std::vector<zg_update> u;
  std::vector<uint8_t> changed;
  rc = delete_found(e, "delete by filter", on_device ? &found : nullptr, &idx, &u, &changed, n_deleted);
  if (rc == ZG_OK) e->log_changes(u, changed);
  return rc;
}

extern "C" int zg_delete_relationships(zg_engine* e, const zg_filter_str* filter, const zg_precondition_str* pre,
                                       uint64_t n_pre, uint64_t* n_deleted) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!filter || (!pre && n_pre)) return fail(ZG_EINVAL, "NULL argument");
  const zg_filter_ex f{*filter, nullptr};
  return delete_all(e, &f, pre_ex(pre, n_pre).data(), n_pre, n_deleted);
}

extern "C" int zg_collect_expired(zg_engine* e, int64_t before_unix, uint64_t* n_removed) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (n_removed) *n_removed = 0;
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  const int64_t clock = e->clock ? e->clock : static_cast<int64_t>(time(nullptr));
  if (before_unix > clock)
    return fail(ZG_EINVAL, "collect expired: before (" + std::to_string(before_unix) + ") is later than the engine's clock (" +
                               std::to_string(clock) + ")");
  // expirations are stored as unsigned 32-bit seconds, and 0 means "never"
  if (!e->schema.has_expiry || before_unix <= 0) return ZG_OK;
  const uint32_t before = static_cast<uint32_t>(std::min<int64_t>(before_unix, 0xFFFFFFFFll));
  std::vector<uint64_t> idx;
  std::vector<zg_tuple> found;
  bool on_device = filters_on_device(e);
  if (on_device) {
    uint64_t count = 0;
    bool too_big = false;
    int rc = ask_devices(e, snapshot_devices(e), Device::kByScan, [&](Device& dev, uint64_t* n, std::vector<zg_tuple>* got, bool* big,
                                                     std::string* err) {
      return dev.match_expired(e->schema, before, n, got, big, err);
    }, &count, &found, &too_big);
    if (rc) return rc;
    on_device = !too_big;
    if (on_device && count == 0) return ZG_OK;
  }
  if (!on_device) {
    e->store.expired(before, &idx);
    ++e->flt_host;
    if (idx.empty()) return ZG_OK;
  }
  // an expiration is not a write: the watch feed records none of these DELETEs
  std::vector<zg_update> u;
  std::vector<uint8_t> changed;
  return delete_found(e, "collect expired", on_device ? &found : nullptr, &idx, &u, &changed, n_removed);
}

extern "C" int zg_retire_unused_names(zg_engine* e, uint64_t* n_retired) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (n_retired) *n_retired = 0;
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  if (e->store.shard_count > 1)
    return fail(ZG_EINVAL, "retire unused names: this engine is one shard of several (zg_config.shard_count) and its store "
                           "does not hold the other shards' relationships");
  // Which ids some relationship of the store names: read from the snapshots when they are the store (every shard of a
  // sharded handle scans its own; replicas hold the same snapshot, so the first device answers), else from the store.
  Store::IdBits keep;
  const bool on_device = filters_on_device(e);
  if (on_device) {
    const uint32_t S = is_handle(e) ? e->n_shards : 1;
    std::vector<Store::IdBits> got(S);
    std::string err;
    if (int rc = on_devices(e, snapshot_devices(e), [&](Device& dev, size_t k, std::string* m) {
          return dev.scan_mentions(e->schema, &got[k], m);
        }, &err))
      return fail(rc == ZG_ENOMEM ? ZG_ECUDA : rc, err);
    keep.swap(got[0]);
    for (uint32_t k = 1; k < S; ++k)
      for (size_t t = 0; t < got[k].size(); ++t) {
        if (keep[t].size() < got[k][t].size()) keep[t].resize(got[k][t].size(), 0);
        for (size_t w = 0; w < got[k][t].size(); ++w) keep[t][w] |= got[k][t][w];
      }
  } else {
    e->store.mentioned(&keep);
  }
  // zg_watch_read renders the retained changes' names when it is called: their ids keep their names
  for (const auto& w : e->watch_log) {
    Store::mark(&keep, e->schema.slots[w.t.rel].type, w.t.res);
    if (w.t.srel != kWildcard) Store::mark(&keep, w.t.stype, w.t.subj);
  }
  const uint64_t n = e->store.retire(keep);
  if (n) {
    // the device mirrors of the names hold the retired records: they are rebuilt by the next device-ingress call
    e->dev.ingress_reset();
    for (auto& r : e->replicas) r->dev.ingress_reset();
    if (on_device) e->retire_device += n;
    else e->retire_host += n;
    ++e->name_epoch;
  }
  if (n_retired) *n_retired = n;
  return ZG_OK;
}

extern "C" int zg_debug_set_resolve_hook(zg_engine* e, void (*hook)(void*), void* arg) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  e->resolve_hook = hook;
  e->resolve_hook_arg = arg;
  return ZG_OK;
}

extern "C" int zg_name_counters(zg_engine* e, uint64_t* out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!out) return fail(ZG_EINVAL, "out is NULL");
  LOCK_NAMES_SHARED(e);
  const Store::NameCounts c = e->store.name_counts();
  out[0] = c.named;
  out[1] = e->store.retired_names;
  out[2] = c.free_ids;
  out[3] = c.extent;
  out[4] = c.arena_bytes;
  out[5] = e->retire_device;
  out[6] = e->retire_host;
  return ZG_OK;
}

extern "C" uint64_t zg_object_capacity(const zg_engine* e, int type_id) {
  NEED_SCHEMA(e, 0);
  LOCK_NAMES_SHARED(e);
  return e->store.capacity(type_id);
}

static std::string tuple_text(const zg_engine* e, const zg_tuple& t) {
  const Schema& sc = e->schema;
  const SlotInfo& rel = sc.slots[t.rel];
  auto obj = [&](int type, uint32_t id) {
    std::string_view n;
    return e->store.name(type, id, &n) ? std::string(n) : std::to_string(id);
  };
  std::string s = sc.types[rel.type].name + ":" + obj(rel.type, t.res) + "#" + rel.name + "@" + sc.types[t.stype].name + ":";
  if (t.srel == kWildcard) return s + "*";
  s += obj(t.stype, t.subj);
  if (t.srel != kNone) s += "#" + sc.slots[t.srel].name;
  return s;
}

extern "C" int zg_read_relationships(zg_engine* e, const zg_filter_str* filter, char* buf, size_t cap, size_t* need,
                                     uint64_t* n_out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!filter) return fail(ZG_EINVAL, "NULL filter");
  const zg_filter_ex f{*filter, nullptr};
  return zg_read_relationships_ex(e, &f, buf, cap, need, n_out);
}

extern "C" int zg_read_relationships_ex(zg_engine* e, const zg_filter_ex* filter, char* buf, size_t cap, size_t* need,
                                        uint64_t* n_out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!filter) return fail(ZG_EINVAL, "NULL filter");
  // Device path: the device lock, then the names lock SHARED, the order every other call uses; checks keep resolving
  // their strings beside the read, and the store's relationship index is never built. Host scan: the names lock
  // exclusively, since match() may (re)build that index.
  std::unique_lock<FairMutex> dl(e->mu, std::defer_lock);
  if (!e->host_only) dl.lock();
  std::shared_lock<std::shared_mutex> shared(e->names, std::defer_lock);
  std::unique_lock<std::shared_mutex> exclusive(e->names, std::defer_lock);
  bool on_device = filters_on_device(e);
  if (on_device) shared.lock();
  else exclusive.lock();
  std::string err;
  Store::Filter f = resolve_filter(e, *filter, &err);
  if (!err.empty()) return fail(ZG_EINVAL, err);
  std::vector<zg_tuple> found;
  if (on_device) {
    uint64_t count = 0;
    bool too_big = false;
    if (int rc = match_on_device(e, f, now_of(e), &count, &found, &too_big)) return rc;
    if (too_big) {  // writers and retirements wait for the device lock held here: f stays resolved
      on_device = false;
      shared.unlock();
      exclusive.lock();
    }
  }
  if (!on_device) {
    std::vector<uint64_t> idx;
    e->store.match(f, now_of(e), &idx);
    count_host(e, f);
    found.reserve(idx.size());
    for (uint64_t i : idx) found.push_back(e->store.tuples[i]);
  }
  std::vector<std::string> lines;
  lines.reserve(found.size());
  for (const zg_tuple& t : found) lines.push_back(tuple_text(e, t));
  std::sort(lines.begin(), lines.end());
  size_t total = 1;
  for (const auto& l : lines) total += l.size() + 1;
  if (need) *need = total;
  if (n_out) *n_out = lines.size();
  if (total > cap || !buf) return ZG_E2BIG;
  size_t w = 0;
  for (const auto& l : lines) {
    std::memcpy(buf + w, l.data(), l.size());
    w += l.size();
    buf[w++] = '\n';
  }
  buf[w] = 0;
  return ZG_OK;
}

// ---- pages: zg_read_relationships_page, zg_delete_relationships_limited ----

// The bytes of a zg_read_cursor. `fp` fingerprints the filter: its type, relation and subject-relation ids as resolved
// against the schema, and the object names as given (a name need not exist, and keeps its meaning across retirements).
struct CursorBits {
  uint16_t version;  // kCursorVersion
  uint16_t has_key;  // 0: the start
  uint32_t schema_gen;
  uint64_t fp;
  PageKey key;
};
static_assert(sizeof(CursorBits) == ZG_READ_CURSOR_BYTES, "zg_read_cursor is CursorBits");
constexpr uint16_t kCursorVersion = 1;
// LookupResources pages (zg_lookup_resources_page*) use the same bytes under their own version, so that a read cursor
// and a lookup cursor are never taken for each other. key.type = the resource type, key.res = the last id returned;
// has_key = kPastIds: after the ids, past a never-written userset subject's own name (the string form's last line).
constexpr uint16_t kLookupCursorVersion = 0x8001;
constexpr uint16_t kPastIds = 2;

static uint64_t filter_fingerprint(const Store::Filter& f, const zg_filter_str& s) {  // f.prefix: mixed in when set
  uint64_t h = 0xcbf29ce484222325ull;
  auto mix = [&](const void* p, size_t n) {
    for (size_t i = 0; i < n; ++i) h = (h ^ static_cast<const uint8_t*>(p)[i]) * 0x100000001b3ull;
  };
  const int32_t ids[6] = {f.res_type, f.rel, f.subj_type, f.subj_wildcard, f.has_srel, f.srel};
  mix(ids, sizeof ids);
  for (const char* str : {s.res_id, s.subj_id}) {
    const size_t n = str ? std::strlen(str) : 0;
    mix(&n, sizeof n);
    if (n) mix(str, n);
  }
  if (!f.prefix.empty()) {  // an unprefixed filter's cursors stay those it always had
    const char tag[] = "prefix";
    mix(tag, sizeof tag);
    const size_t n = f.prefix.size();
    mix(&n, sizeof n);
    mix(f.prefix.data(), n);
  }
  return h;
}

// version: kCursorVersion, or kLookupCursorVersion for a LookupResources page; has_key: what a non-null key holds
static zg_read_cursor make_cursor(const zg_engine* e, uint64_t fp, const PageKey* key, uint16_t version = kCursorVersion,
                                  uint16_t has_key = 1) {
  CursorBits c{};
  c.version = version;
  c.has_key = key ? has_key : 0;
  c.schema_gen = e->schema_gen;
  c.fp = fp;
  if (key) c.key = *key;
  zg_read_cursor out;
  std::memcpy(out.opaque, &c, sizeof c);
  return out;
}

// The first `want` matches of f at clock `now` after *after in the page order, with their expirations, from the
// resident snapshot(s). A sharded handle asks every shard (or the resource's owner) for its own first `want` and merges
// them; replicas hold the same snapshot, so the first device answers. Counts the page in zg_page_counters and the
// filter in zg_filter_counters. *too_big: see Device::page_filter. Caller holds e->mu and e->names (shared is enough)
// and has seen filters_on_device.
static int page_on_device(zg_engine* e, const Store::Filter& f, uint32_t now, const PageKey* after, uint64_t want,
                          std::vector<zg_tuple>* found, std::vector<uint32_t>* exp, bool* too_big) {
  const uint32_t S = is_handle(e) ? e->n_shards : 1;
  std::vector<std::vector<zg_tuple>> got(S);
  std::vector<std::vector<uint32_t>> got_exp(S);
  std::vector<Device::PageStats> st(S);
  std::vector<char> big(S, 0);
  std::string err;
  PrefixBits px;
  const bool has_prefix = !f.prefix.empty();
  if (has_prefix) {
    if (int rc = prefix_on_device(e, f, &px, too_big)) return rc;
    if (*too_big) return ZG_OK;
  }
  if (int rc = on_devices(e, snapshot_devices(e, &f), [&](Device& dev, size_t k, std::string* m) {
        bool b = false;
        const int prc = dev.page_filter(e->schema, f, now, after, want, &got[k], &got_exp[k], &st[k], &b, m,
                                        has_prefix ? &px : nullptr);
        big[k] = b;
        return prc;
      }, &err))
    return fail(rc == ZG_ENOMEM ? ZG_ECUDA : rc, err);
  *too_big = false;
  for (uint32_t k = 0; k < S; ++k) *too_big = *too_big || big[k];
  if (*too_big) return ZG_OK;
  found->clear();
  exp->clear();
  if (S == 1) {
    found->swap(got[0]);
    exp->swap(got_exp[0]);
  } else {  // every shard's list is in K order: merge and cut
    std::vector<std::pair<PageKey, std::pair<uint32_t, uint32_t>>> keys;
    for (uint32_t k = 0; k < S; ++k)
      for (uint32_t i = 0; i < got[k].size(); ++i) keys.push_back({page_key(e->schema, got[k][i]), {k, i}});
    std::sort(keys.begin(), keys.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    if (keys.size() > want) keys.resize(want);
    for (const auto& x : keys) {
      found->push_back(got[x.second.first][x.second.second]);
      exp->push_back(got_exp[x.second.first][x.second.second]);
    }
  }
  ++e->pg_device;
  for (const auto& x : st) {
    e->pg_scanned += x.scanned;
    e->pg_launches += x.launches;
    e->px_launches += x.list_launches;
  }
  if (has_prefix) ++e->px_device;
  ++e->flt_device;
  ++e->flt_shape[Device::filter_shape(f)];
  e->flt_returned += found->size();
  return ZG_OK;
}

// The host path of a page: Store::page. Caller holds e->names exclusively (match() may build the index).
static void page_on_host(zg_engine* e, const Store::Filter& f, uint32_t now, const PageKey* after, uint64_t want,
                         std::vector<zg_tuple>* found, std::vector<uint32_t>* exp) {
  std::vector<uint64_t> idx;
  e->store.page(f, now, after, want, &idx);
  found->clear();
  exp->clear();
  for (uint64_t i : idx) {
    found->push_back(e->store.tuples[i]);
    exp->push_back(e->store.expires[i]);
  }
  ++e->pg_host;
  count_host(e, f);
}

extern "C" int zg_read_relationships_page(zg_engine* e, const zg_filter_str* filter, uint64_t limit, const zg_read_cursor* after,
                                          char* buf, size_t cap, size_t* need, uint64_t* n_out, uint32_t* expires,
                                          zg_read_cursor* cursors, zg_read_cursor* next, int32_t* more) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!filter) return fail(ZG_EINVAL, "NULL filter");
  const zg_filter_ex f{*filter, nullptr};
  return zg_read_relationships_page_ex(e, &f, limit, after, buf, cap, need, n_out, expires, cursors, next, more);
}

extern "C" int zg_read_relationships_page_ex(zg_engine* e, const zg_filter_ex* filter, uint64_t limit, const zg_read_cursor* after,
                                             char* buf, size_t cap, size_t* need, uint64_t* n_out, uint32_t* expires,
                                             zg_read_cursor* cursors, zg_read_cursor* next, int32_t* more) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!filter) return fail(ZG_EINVAL, "NULL filter");
  if (limit == 0) return fail(ZG_EINVAL, "page limit must be at least 1 (zg_read_relationships reads without one)");
  // the locks of zg_read_relationships
  std::unique_lock<FairMutex> dl(e->mu, std::defer_lock);
  if (!e->host_only) dl.lock();
  std::shared_lock<std::shared_mutex> shared(e->names, std::defer_lock);
  std::unique_lock<std::shared_mutex> exclusive(e->names, std::defer_lock);
  bool on_device = filters_on_device(e);
  if (on_device) shared.lock();
  else exclusive.lock();
  std::string err;
  Store::Filter f = resolve_filter(e, *filter, &err);
  if (!err.empty()) return fail(ZG_EINVAL, err);
  const uint64_t fp = filter_fingerprint(f, filter->f);
  CursorBits c{};
  if (after) {
    std::memcpy(&c, after->opaque, sizeof c);
    if (c.version != kCursorVersion || c.has_key > 1)
      return fail(ZG_EINVAL, "read cursor: not a cursor of this engine");
    if (c.schema_gen != e->schema_gen || c.fp != fp)
      return fail(ZG_EINVAL, "read cursor: it was made for another filter or under another schema");
  }
  const PageKey* from = after && c.has_key ? &c.key : nullptr;
  // at most every relationship of the store matches: a larger limit asks the kernels for nothing more
  const uint64_t want = std::min<uint64_t>(limit, e->store.size()) + 1;
  std::vector<zg_tuple> found;
  std::vector<uint32_t> exp;
  if (on_device) {
    bool too_big = false;
    if (int rc = page_on_device(e, f, now_of(e), from, want, &found, &exp, &too_big)) return rc;
    if (too_big) {  // as in zg_read_relationships: writers wait for the device lock held here, f stays resolved
      on_device = false;
      shared.unlock();
      exclusive.lock();
    }
  }
  if (!on_device) page_on_host(e, f, now_of(e), from, want, &found, &exp);
  const bool has_more = found.size() > limit;
  if (has_more) {
    found.resize(limit);
    exp.resize(limit);
  }
  std::vector<std::string> lines;
  lines.reserve(found.size());
  size_t total = 1;
  for (const zg_tuple& t : found) {
    lines.push_back(tuple_text(e, t));
    total += lines.back().size() + 1;
  }
  if (need) *need = total;
  if (n_out) *n_out = lines.size();
  if (total > cap || !buf) return ZG_E2BIG;
  size_t w = 0;
  for (size_t i = 0; i < lines.size(); ++i) {
    std::memcpy(buf + w, lines[i].data(), lines[i].size());
    w += lines[i].size();
    buf[w++] = '\n';
    if (expires) expires[i] = exp[i];
    if (cursors) {
      const PageKey k = page_key(e->schema, found[i]);
      cursors[i] = make_cursor(e, fp, &k);
    }
  }
  buf[w] = 0;
  if (next) {
    if (found.empty()) *next = make_cursor(e, fp, from);
    else {
      const PageKey k = page_key(e->schema, found.back());
      *next = make_cursor(e, fp, &k);
    }
  }
  if (more) *more = has_more;
  return ZG_OK;
}

extern "C" int zg_delete_relationships_limited(zg_engine* e, const zg_filter_str* filter, const zg_precondition_str* pre,
                                               uint64_t n_pre, uint64_t limit, int allow_partial, uint64_t* n_deleted,
                                               int32_t* partial) {
  if (partial) *partial = 0;
  if (limit == 0) return zg_delete_relationships(e, filter, pre, n_pre, n_deleted);
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!filter || (!pre && n_pre)) return fail(ZG_EINVAL, "NULL argument");
  const zg_filter_ex f{*filter, nullptr};
  return zg_delete_relationships_limited_ex(e, &f, pre_ex(pre, n_pre).data(), n_pre, limit, allow_partial, n_deleted, partial);
}

extern "C" int zg_delete_relationships_limited_ex(zg_engine* e, const zg_filter_ex* filter, const zg_precondition_ex* pre,
                                                  uint64_t n_pre, uint64_t limit, int allow_partial, uint64_t* n_deleted,
                                                  int32_t* partial) {
  if (partial) *partial = 0;
  if (limit == 0) return delete_all(e, filter, pre, n_pre, n_deleted);
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!filter || (!pre && n_pre)) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  std::string err;
  Store::Filter f = resolve_filter(e, *filter, &err);
  if (!err.empty()) return fail(ZG_EINVAL, err);
  int rc = check_preconditions(e, pre, n_pre);
  if (rc) return rc;
  // the first limit + 1 matches in the page order, expired ones included (clock 0): is there more than the limit?
  const uint64_t want = std::min<uint64_t>(limit, e->store.size()) + 1;
  std::vector<zg_tuple> found;
  std::vector<uint32_t> exp;
  bool on_device = filters_on_device(e);
  if (on_device) {
    bool too_big = false;
    if ((rc = page_on_device(e, f, 0, nullptr, want, &found, &exp, &too_big))) return rc;
    on_device = !too_big;
  }
  if (!on_device) page_on_host(e, f, 0, nullptr, want, &found, &exp);
  const bool cut = found.size() > limit;
  if (cut && !allow_partial)  // the text of SpiceDB's DeleteRelationships
    return fail(ZG_EPRECOND, "found more than " + std::to_string(limit) +
                                 " relationships to be deleted and partial deletion was not requested");
  if (cut) found.resize(limit);
  std::vector<uint64_t> idx;
  std::vector<zg_update> u;
  std::vector<uint8_t> changed;
  rc = delete_found(e, "delete by filter", &found, &idx, &u, &changed, n_deleted);
  if (rc == ZG_OK) {
    e->log_changes(u, changed);
    if (partial) *partial = cut;
  }
  return rc;
}

extern "C" int zg_page_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  const uint64_t c[4] = {e->pg_device.load(), e->pg_host.load(), e->pg_scanned.load(), e->pg_launches.load()};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_prefix_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  const uint64_t c[6] = {e->px_device.load(), e->px_host.load(), e->px_names.load(), e->px_matched.load(),
                         e->px_launches.load(), e->px_syncs.load()};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_watch_read(zg_engine* e, uint64_t since_revision, const char* res_type, char* buf, size_t cap,
                             size_t* need, uint64_t* n_out, uint64_t* through_revision) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  LOCK_DEVICE(e);  // the change log is appended under the device lock
  LOCK_NAMES_SHARED(e);
  int want = -1;
  if (res_type && *res_type) {
    want = e->schema.type_id(res_type);
    if (want < 0) return fail(ZG_EINVAL, std::string("object definition `") + res_type + "` not found");
  }
  if (since_revision < e->watch_floor)
    return fail(ZG_EPRECOND, "watch: revision " + std::to_string(since_revision) + " is older than the retained feed (" +
                                 std::to_string(e->watch_floor) + ")");
  static const char* kOp[] = {"TOUCH", "CREATE", "DELETE"};
  std::string out;
  uint64_t n = 0;
  // entries are in revision order: binary search for the first one after `since`
  auto it = std::partition_point(e->watch_log.begin(), e->watch_log.end(),
                                 [&](const zg_engine::WatchEntry& w) { return w.revision <= since_revision; });
  for (; it != e->watch_log.end(); ++it) {
    if (want >= 0 && e->schema.slots[it->t.rel].type != want) continue;
    out += std::to_string(it->revision);
    out += ' ';
    out += kOp[it->op];
    out += ' ';
    out += tuple_text(e, it->t);
    if (it->expires_at && it->op != ZG_OP_DELETE) out += " " + std::to_string(it->expires_at);
    out += '\n';
    ++n;
  }
  if (need) *need = out.size() + 1;
  if (n_out) *n_out = n;
  if (through_revision) *through_revision = e->revision;
  if (out.size() + 1 > cap || !buf) return ZG_E2BIG;
  std::memcpy(buf, out.data(), out.size());
  buf[out.size()] = 0;
  return ZG_OK;
}

// ---- hot path ------------------------------------------------------------------------

// Makes pending writes visible before a string entry point resolves against them. Takes both locks only when
// there is something to publish; call it with NO lock held.
static int publish_if_needed(zg_engine* e) {
  if (int rc = refuse(e, Call::kCheckGroup)) return rc;
  if (!e->dirty.load() && e->dev.snap) return ZG_OK;
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  if (e->dirty.load() || !e->dev.snap) return publish_locked(e);
  return ZG_OK;
}

// The checks of one run of the handle's check protocol: shard k brings n[k] items at items[k] and gets their codes at
// out[k], in the same order. Host (pinned) or that shard's device memory, both.
struct ShardLists {
  std::vector<const zg_check*> items;
  std::vector<uint64_t> n;
  std::vector<uint8_t*> out;
};

// Lays out the inboxes of one exchange among the S shards from its count matrix (counts[k * S + d]: entries shard k
// sends to shard d), for destinations d < n_dest: in d's inbox, shard k's entries follow those of the lower shards, and
// tab[k] says where shard k writes them. inbox(d, n) returns d's inbox grown to n entries, or nullptr (then false).
template <class Inbox>
static bool lay_out_inboxes(uint32_t S, uint32_t n_dest, const std::vector<uint64_t>& counts, std::vector<PeerTable>* tab,
                            Inbox&& inbox) {
  for (uint32_t d = 0; d < n_dest; ++d) {
    uint64_t at = 0;
    for (uint32_t k = 0; k < S; ++k) {
      (*tab)[k].base[d] = at;
      at += counts[size_t(k) * S + d];
    }
    void* p = inbox(d, at);
    if (!p) return false;
    for (uint32_t k = 0; k < S; ++k) (*tab)[k].p[d] = p;
  }
  return true;
}

// The levels of dist.DeviceShardedChecker.check_bulk, driven in this process. Every shard routes its list to the
// owners. Per level, every shard writes its queries straight into the owners' inboxes (where, the host computes from
// every shard's counts: the level's one round trip), each owner's pass starts when the shards delivering to it are
// done (events, not host waits), and the values are folded back level by level where their owners left them.
// *overflow: a pass raised more sub-queries than its buffer holds; nothing is answered. no_wildcards: every pass of
// every shard, the sub-queries' included, sees no wildcard relationship (LookupSubjects' second verification).
static int sharded_levels(zg_engine* e, const ShardLists& L, PeerCounts* pc, bool no_wildcards, bool* overflow_out,
                          std::string* err) {
  const uint32_t S = e->n_shards;
  *overflow_out = false;
  std::vector<uint64_t> counts(size_t(S) * S, 0);  // [k * S + d]: queries shard k sends to shard d this level
  const uint32_t now = now_of(e);
  ++pc->round_trips;
  if (int rc = on_devices(e, kEveryDevice, [&](Device& dev, size_t k, std::string* m) {
        dev.now = now;
        return dev.peer_begin(L.items[k], L.n[k], &counts[k * S], m);
      }, err))
    return rc;
  std::vector<PeerTable> tab(S);
  std::vector<cudaEvent_t> wait(S);
  auto events = [&](int level) {
    for (uint32_t k = 0; k < S; ++k) wait[k] = shard(e, k).peer_event(level);
  };
  std::vector<uint64_t> nsub(S);
  std::vector<char> overflow(S);
  int level = 0;
  for (;; ++level) {
    uint64_t total = 0;
    if (!lay_out_inboxes(S, S, counts, &tab, [&](uint32_t d, uint64_t n) {
          total += n;
          return shard(e, d).peer_inbox(level, n, err);
        }))
      return ZG_ENOMEM;
    if (total == 0) break;
    if (level > ZG_MAX_DEPTH + 1) {
      *err = "sub-query passes exceeded the depth cap";
      return ZG_ECUDA;
    }
    if (int rc = on_devices(e, kEveryDevice, [&](Device& dev, size_t k, std::string* m) {
          return dev.peer_scatter(level, tab[k], m);
        }, err))
      return rc;
    events(level);
    ++pc->round_trips;
    pc->levels = std::max<uint64_t>(pc->levels, static_cast<uint64_t>(level) + 1);
    if (int rc = on_devices(e, kEveryDevice, [&](Device& dev, size_t k, std::string* m) {
          bool o = false;
          const int prc = dev.peer_pass(level, wait, &nsub[k], &counts[k * S], &o, no_wildcards, m);
          overflow[k] = o;
          return prc;
        }, err))
      return rc;
    if (std::find(overflow.begin(), overflow.end(), 1) != overflow.end()) {
      *overflow_out = true;
      return ZG_OK;
    }
    for (uint32_t k = 0; k < S; ++k) pc->subqueries += nsub[k];
  }
  // values back: the deepest pass raised nothing; every shallower level folds in its children's values
  auto values_of = [&](int lv) {
    for (uint32_t d = 0; d < S; ++d) {
      tab[0].p[d] = const_cast<uint8_t*>(shard(e, d).peer_values(lv));
      tab[0].base[d] = 0;
    }
    events(lv);
  };
  for (int lv = level - 2; lv >= 0; --lv) {
    values_of(lv + 1);
    if (int rc = on_devices(e, kEveryDevice, [&](Device& dev, size_t, std::string* m) {
          return dev.peer_fold(lv, tab[0], wait, m);
        }, err))
      return rc;
  }
  values_of(0);
  ++pc->round_trips;
  return on_devices(e, kEveryDevice, [&](Device& dev, size_t k, std::string* m) {
    return dev.peer_finish(tab[0], wait, L.out[k], m);
  }, err);
}

// sharded_levels, and on overflow the same in halves (checks are independent): the first half of the items taken in
// shard order, then the rest. Where an item starts does not change where it is evaluated (at its owner).
static int run_sharded_lists(zg_engine* e, const ShardLists& L, PeerCounts* pc, bool no_wildcards, std::string* err) {
  bool overflow = false;
  if (int rc = sharded_levels(e, L, pc, no_wildcards, &overflow, err)) return rc;
  if (!overflow) return ZG_OK;
  uint64_t n = 0;
  for (uint64_t m : L.n) n += m;
  if (n < 2) {
    *err = "sub-query buffer overflow on a single check: raise zg_config.subquery_capacity";
    return ZG_ENOMEM;
  }
  ++e->dev.split_batches;
  ShardLists a = L, b = L;
  uint64_t h = n / 2;
  for (size_t k = 0; k < L.n.size(); ++k) {
    a.n[k] = std::min(h, L.n[k]);
    h -= a.n[k];
    b.n[k] = L.n[k] - a.n[k];
    b.items[k] += a.n[k];
    b.out[k] += a.n[k];
  }
  if (int rc = run_sharded_lists(e, a, pc, no_wildcards, err)) return rc;
  return run_sharded_lists(e, b, pc, no_wildcards, err);
}

// n checks in host memory (out: their codes): shard k brings the slice dist.shard_bounds gives it.
static int run_sharded(zg_engine* e, const zg_check* items, uint64_t n, uint8_t* out, PeerCounts* pc, std::string* err) {
  const uint32_t S = e->n_shards;
  auto lo = [&](uint32_t k) { return k * (n / S) + std::min<uint64_t>(k, n % S); };
  ShardLists L;
  for (uint32_t k = 0; k < S; ++k) {
    L.items.push_back(items + lo(k));
    L.n.push_back(lo(k + 1) - lo(k));
    L.out.push_back(out + lo(k));
  }
  return run_sharded_lists(e, L, pc, false, err);
}

// Answers one group of queued requests; the caller holds the device lock.
static int run_group(zg_engine* e, const std::vector<BatchReq*>& group, std::string* err) {
  if (int rc = refuse(e, Call::kCheckGroup, err)) return rc;
  bool published = e->dev.snap != nullptr;
  for (uint32_t k = 1; k < e->n_shards; ++k) published = published && shard(e, k).snap;
  if (!published) {
    *err = "no snapshot published (call zg_publish)";
    return ZG_ENOSNAPSHOT;
  }
  uint64_t total = 0;
  for (BatchReq* r : group) total += r->n;
  if (is_handle(e)) {
    const size_t bytes = total * (sizeof(zg_check) + 1);  // the items, then their answers
    if (e->group_pin_cap < bytes) {
      if (e->group_pin) cudaFreeHost(e->group_pin);
      e->group_pin = nullptr;
      e->group_pin_cap = 0;
      if (cudaMallocHost(&e->group_pin, bytes) == cudaSuccess) e->group_pin_cap = bytes;
      else cudaGetLastError();
    }
    if (!e->group_pin) {
      *err = "out of pinned host memory (sharded handle staging)";
      return ZG_ENOMEM;
    }
    zg_check* items = static_cast<zg_check*>(e->group_pin);
    uint64_t off = 0;
    for (BatchReq* r : group) {
      std::memcpy(items + off, r->items, r->n * sizeof(zg_check));
      off += r->n;
    }
    uint8_t* answers = reinterpret_cast<uint8_t*>(items + total);
    e->last_group = PeerCounts();
    const int rc = run_sharded(e, items, total, answers, &e->last_group, err);
    off = 0;
    for (BatchReq* r : group) {
      if (!rc) std::memcpy(r->out, answers + off, r->n);
      off += r->n;
    }
    if (group.size() > 1) {
      ++e->dev.coalesced_launches;
      e->dev.coalesced_requests += group.size();
    }
    return rc;
  }
  std::vector<Device::HostReq> reqs;
  reqs.reserve(group.size());
  for (BatchReq* r : group) reqs.push_back({r->items, r->n, r->out});
  const size_t nd = 1 + e->replicas.size();
  if (nd == 1 || total < nd * 4096) {
    e->dev.now = now_of(e);
    return e->dev.check_host_multi(reqs, err);
  }
  // replicas: every device answers a contiguous slice of the group's items
  std::vector<std::vector<Device::HostReq>> part(nd);
  const uint64_t per = (total + nd - 1) / nd;
  size_t d = 0;
  uint64_t room = per;
  for (const auto& r : reqs) {
    uint64_t off = 0;
    while (off < r.n) {
      const uint64_t take = std::min(room, r.n - off);
      part[d].push_back({r.items + off, take, r.out + off});
      off += take;
      room -= take;
      if (room == 0 && d + 1 < nd) {
        ++d;
        room = per;
      }
    }
  }
  const uint32_t now = now_of(e);
  return on_devices(e, kEveryDevice, [&](Device& dev, size_t i, std::string* m) {
    dev.now = now;
    return part[i].empty() ? ZG_OK : dev.check_host_multi(part[i], m);
  }, err);
}

extern "C" int zg_check_bulk(zg_engine* e, const zg_check* items, uint64_t n, uint8_t* out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if ((!items || !out) && n) return fail(ZG_EINVAL, "NULL argument");
  if (n == 0) return ZG_OK;
  BatchReq me;
  me.items = items;
  me.n = n;
  me.out = out;
  e->batcher.submit(
      &me, e->mu,
      [](const std::vector<BatchReq*>& queue) {  // as many callers as fit one launch, and always the first
        uint64_t total = queue[0]->n;
        size_t take = 1;
        while (take < queue.size() && total + queue[take]->n <= kMaxItemsPerLaunch) total += queue[take++]->n;
        return take;
      },
      [e](const std::vector<BatchReq*>& group) {
        std::string err;
        const int rc = run_group(e, group, &err);
        for (BatchReq* r : group) {
          r->rc = rc;
          r->err = err;
        }
      });
  return me.rc ? fail(me.rc, me.err) : ZG_OK;
}

extern "C" int zg_check_bulk_device(zg_engine* e, const zg_check* d_items, uint64_t n, uint8_t* d_out, void* stream) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if ((!d_items || !d_out) && n) return fail(ZG_EINVAL, "NULL argument");
  std::lock_guard<FairMutex> g(e->mu);
  if (int rc = refuse(e, Call::kDeviceChecks)) return rc;
  e->dev.now = now_of(e);
  std::string err;
  int rc = e->dev.check_device(d_items, n, d_out, static_cast<cudaStream_t>(stream), true, nullptr, &err);
  return rc ? fail(rc, err) : ZG_OK;
}

extern "C" int zg_count_alg_bytes(zg_engine* e, const zg_check* items, uint64_t n, uint64_t* bytes) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!items || !bytes) return fail(ZG_EINVAL, "NULL argument");
  std::lock_guard<FairMutex> g(e->mu);
  if (int rc = refuse(e, Call::kDeviceBuffers)) return rc;
  e->dev.now = now_of(e);
  std::string err;
  void *d_in = nullptr, *d_out = nullptr;
  if (cudaMalloc(&d_in, n * sizeof(zg_check)) != cudaSuccess || cudaMalloc(&d_out, n ? n : 1) != cudaSuccess) {
    if (d_in) cudaFree(d_in);
    return fail(ZG_ENOMEM, "out of device memory");
  }
  cudaMemcpy(d_in, items, n * sizeof(zg_check), cudaMemcpyHostToDevice);
  uint64_t b = 0;
  int rc = e->dev.check_device(static_cast<zg_check*>(d_in), n, static_cast<uint8_t*>(d_out), e->dev.stream, true, &b, &err);
  cudaFree(d_in);
  cudaFree(d_out);
  if (rc) return fail(rc, err);
  *bytes = b;
  return ZG_OK;
}

extern "C" int zg_phase_clocks(zg_engine* e, uint64_t cycles[5]) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!cycles) return fail(ZG_EINVAL, "NULL argument");
  std::lock_guard<FairMutex> g(e->mu);
  if (int rc = refuse(e, Call::kDevice)) return rc;
  std::string err;
  const int rc = e->dev.read_phase_clocks(cycles, &err);
  return rc ? fail(rc, err) : ZG_OK;
}

// Resolve a CHECK item without interning anything (query strings must not grow the store).
// The items of one bulk call mostly repeat their literal fields -- a post-filter sends one template
// per list item, so type, permission and subject are constant and only the resource id varies
// (pkg/authz/postfilter.go:88-110; "low-hanging fruit" in pkg/rules/rules.go:1015-1017) -- so the
// schema lookups and the subject lookup of the previous item are reused when the strings repeat.
struct ResolveMemo {
  struct SchemaPart {  // (res_type, relation, subj_type, subj_rel) -> slots
    std::string res_type, relation, subj_type, subj_rel;
    int rt = -1, st = -1, perm = -1;
    uint16_t srel = kNone;
    bool ok = false, used = false;
  };
  static constexpr int kWays = 4;  // a bulk request interleaves a handful of templates at most
  SchemaPart parts[kWays];
  int last = 0, next = 0;
  std::string subj_id;  // subject of the previous item
  int subj_st = -1;
  uint32_t su = ZG_NO_OBJECT;
};

static inline bool same(const std::string& a, const char* b) { return std::strcmp(a.c_str(), b) == 0; }

static const ResolveMemo::SchemaPart& resolve_schema_part(const Schema& sc, const zg_rel_str& r, const char* srel_s,
                                                          ResolveMemo* m) {
  for (int k = 0; k < ResolveMemo::kWays; ++k) {
    const int w = (m->last + k) % ResolveMemo::kWays;
    const ResolveMemo::SchemaPart& p = m->parts[w];
    if (p.used && same(p.res_type, r.res_type) && same(p.relation, r.relation) && same(p.subj_type, r.subj_type) &&
        same(p.subj_rel, srel_s)) {
      m->last = w;
      return p;
    }
  }
  const int w = m->next;
  m->next = (m->next + 1) % ResolveMemo::kWays;
  ResolveMemo::SchemaPart& p = m->parts[w];
  p.res_type = r.res_type;
  p.relation = r.relation;
  p.subj_type = r.subj_type;
  p.subj_rel = srel_s;
  p.used = true;
  p.ok = false;
  p.srel = kNone;
  p.rt = sc.type_id(r.res_type);
  p.st = sc.type_id(r.subj_type);
  if (p.rt >= 0 && p.st >= 0) {
    p.perm = sc.slot_id(p.rt, r.relation);
    const int sr = *srel_s ? sc.slot_id(p.st, srel_s) : 0;
    if (p.perm >= 0 && sr >= 0) {
      if (*srel_s) p.srel = static_cast<uint16_t>(sr);
      p.ok = true;
    }
  }
  m->last = w;
  return p;
}

static void resolve_check(const zg_engine* e, const zg_rel_str& r, zg_check* c, ResolveMemo* m) {
  c->res = ZG_NO_OBJECT;
  c->subj = ZG_NO_OBJECT - 1;
  c->perm = kNone;  // invalid -> ZG_ITEM_ERROR
  c->stype = 0;
  c->srel = kNone;
  c->flags = 0;
  if (!r.res_type || !r.res_id || !r.relation || !r.subj_type || !r.subj_id) return;
  const ResolveMemo::SchemaPart& p = resolve_schema_part(e->schema, r, none_rel(r.subj_rel) ? "" : r.subj_rel, m);
  if (!p.ok) return;
  const int rt = p.rt, st = p.st;
  c->srel = p.srel;
  c->stype = static_cast<uint16_t>(st);
  c->res = e->store.find(rt, r.res_id, std::strlen(r.res_id));
  if (!(m->subj_st == st && same(m->subj_id, r.subj_id))) {
    m->subj_id = r.subj_id;
    m->su = e->store.find(st, r.subj_id, m->subj_id.size());
    m->subj_st = st;
  }
  uint32_t su = m->su;
  // two never-written names that are the same object must still compare equal
  if (su == ZG_NO_OBJECT) su = (c->res == ZG_NO_OBJECT && rt == st && std::strcmp(r.res_id, r.subj_id) == 0)
                                   ? ZG_NO_OBJECT : ZG_NO_OBJECT - 1;
  c->subj = su;
  c->perm = static_cast<uint16_t>(p.perm);
}

static void resolve_checks_locked(const zg_engine* e, const zg_rel_str* items, uint64_t n, zg_check* out) {
  auto run = [&](uint64_t b, uint64_t en) {
    ResolveMemo memo;
    for (uint64_t i = b; i < en; ++i) resolve_check(e, items[i], &out[i], &memo);
  };
  // Resolution only reads the schema and the interning tables (the engine lock is held), so a large
  // batch is split over host threads; below ~16k items one thread finishes before others would start.
  constexpr uint64_t kPerThread = 8192;
  unsigned hw = std::thread::hardware_concurrency();
  uint64_t nt = std::min<uint64_t>({n / kPerThread, hw ? hw : 1u, 16u});
  if (nt < 2) return run(0, n);
  std::vector<std::thread> th;
  th.reserve(nt - 1);
  const uint64_t per = (n + nt - 1) / nt;
  for (uint64_t t = 1; t < nt; ++t) th.emplace_back(run, std::min(n, t * per), std::min(n, (t + 1) * per));
  run(0, std::min(n, per));
  for (auto& x : th) x.join();
}

extern "C" int zg_resolve_checks(zg_engine* e, const zg_rel_str* items, uint64_t n, zg_check* out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if ((!items || !out) && n) return fail(ZG_EINVAL, "NULL argument");
  LOCK_NAMES_SHARED(e);
  resolve_checks_locked(e, items, n, out);
  return ZG_OK;
}

static int resolve_packed_locked(zg_engine* e, const char* res_type, const char* relation, const char* subj_type,
                                 const char* subj_rel, const char* res_ids, const uint32_t* res_off, const char* subj_ids,
                                 const uint32_t* subj_off, uint64_t n, zg_check* out) {
  for (uint64_t i = 0; i < n; ++i)
    if (res_off[i] > res_off[i + 1] || (subj_off && subj_off[i] > subj_off[i + 1]))
      return fail(ZG_EINVAL, "offsets must not decrease");
  // the literal fields once (same rules as resolve_check)
  ResolveMemo memo;
  zg_check base;
  const zg_rel_str proto{res_type, "", relation, subj_type, subj_off ? "" : subj_ids, subj_rel};
  resolve_check(e, proto, &base, &memo);
  const ResolveMemo::SchemaPart& part = memo.parts[memo.last];
  const bool ok = base.perm != kNone;
  const size_t one_len = subj_off ? 0 : std::strlen(subj_ids);
  auto run = [&](uint64_t b, uint64_t en) {
    for (uint64_t i = b; i < en; ++i) {
      out[i] = base;
      if (!ok) continue;  // unknown type / relation: answers ZG_ITEM_ERROR like the string path
      const char* rid = res_ids + res_off[i];
      const size_t rl = res_off[i + 1] - res_off[i];
      const char* sid = subj_off ? subj_ids + subj_off[i] : subj_ids;
      const size_t sl = subj_off ? subj_off[i + 1] - subj_off[i] : one_len;
      const uint32_t res = e->store.find(part.rt, rid, rl);
      uint32_t su = subj_off ? e->store.find(part.st, sid, sl) : memo.su;
      if (su == ZG_NO_OBJECT)
        su = (res == ZG_NO_OBJECT && part.rt == part.st && rl == sl && std::memcmp(rid, sid, rl) == 0) ? ZG_NO_OBJECT
                                                                                                       : ZG_NO_OBJECT - 1;
      out[i].res = res;
      out[i].subj = su;
    }
  };
  constexpr uint64_t kPerThread = 16384;
  const unsigned hw = std::thread::hardware_concurrency();
  const uint64_t nt = std::min<uint64_t>({n / kPerThread, hw ? hw : 1u, 16u});
  if (nt < 2) {
    run(0, n);
    return ZG_OK;
  }
  std::vector<std::thread> th;
  const uint64_t per = (n + nt - 1) / nt;
  for (uint64_t t = 1; t < nt; ++t) th.emplace_back(run, std::min(n, t * per), std::min(n, (t + 1) * per));
  run(0, std::min(n, per));
  for (auto& x : th) x.join();
  return ZG_OK;
}

#define PACKED_ARGS_OK() \
  (res_type && relation && subj_type && (n == 0 || (res_ids && res_off && subj_ids && out)))

extern "C" int zg_resolve_checks_packed(zg_engine* e, const char* res_type, const char* relation, const char* subj_type,
                                        const char* subj_rel, const char* res_ids, const uint32_t* res_off,
                                        const char* subj_ids, const uint32_t* subj_off, uint64_t n, zg_check* out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!PACKED_ARGS_OK()) return fail(ZG_EINVAL, "NULL argument");
  if (n == 0) return ZG_OK;
  LOCK_NAMES_SHARED(e);
  return resolve_packed_locked(e, res_type, relation, subj_type, subj_rel, res_ids, res_off, subj_ids, subj_off, n, out);
}

static int check_bulk_packed_once(zg_engine* e, const char* res_type, const char* relation, const char* subj_type,
                                  const char* subj_rel, const char* res_ids, const uint32_t* res_off, const char* subj_ids,
                                  const uint32_t* subj_off, uint64_t n, uint8_t* out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!PACKED_ARGS_OK()) return fail(ZG_EINVAL, "NULL argument");
  if (n == 0) return ZG_OK;
  std::vector<zg_check> c(n);
  {
    int rc = publish_if_needed(e);
    if (rc) return rc;
    LOCK_NAMES_SHARED(e);
    rc = resolve_packed_locked(e, res_type, relation, subj_type, subj_rel, res_ids, res_off, subj_ids, subj_off, n, c.data());
    if (rc) return rc;
  }
  if (e->resolve_hook) e->resolve_hook(e->resolve_hook_arg);
  return zg_check_bulk(e, c.data(), n, out);
}

extern "C" int zg_check_bulk_packed(zg_engine* e, const char* res_type, const char* relation, const char* subj_type,
                                    const char* subj_rel, const char* res_ids, const uint32_t* res_off, const char* subj_ids,
                                    const uint32_t* subj_off, uint64_t n, uint8_t* out) {
  return with_stable_names(e, [&] {
    return check_bulk_packed_once(e, res_type, relation, subj_type, subj_rel, res_ids, res_off, subj_ids, subj_off,
                                  n, out);
  });
}

static int check_bulk_str_once(zg_engine* e, const zg_rel_str* items, uint64_t n, uint8_t* out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if ((!items || !out) && n) return fail(ZG_EINVAL, "NULL argument");
  std::vector<zg_check> c(n);
  {
    int rc = publish_if_needed(e);
    if (rc) return rc;
    LOCK_NAMES_SHARED(e);
    resolve_checks_locked(e, items, n, c.data());
  }
  // The launch goes through the batcher like any zg_check_bulk call, after the names lock is released: concurrent
  // string callers -- one goroutine per rule check in the proxy, pkg/authz/check.go:77-93 -- share launches too. Ids
  // keep their names across writes; a retirement in between is caught by zg_check_bulk_str (with_stable_names).
  if (e->resolve_hook) e->resolve_hook(e->resolve_hook_arg);
  return zg_check_bulk(e, c.data(), n, out);
}

extern "C" int zg_check_bulk_str(zg_engine* e, const zg_rel_str* items, uint64_t n, uint8_t* out) {
  return with_stable_names(e, [&] { return check_bulk_str_once(e, items, n, out); });
}

// ---- device ingress: packed ids resolved on the GPU against a mirror of the interned names ----------
//
// Each call takes the device lock, then the names lock shared: the mirror's sync (Device::ingress_sync) and the
// resolve kernel never race a writer or each other, and the call returns after its GPU work has completed.

// The literal fields, resolved once exactly as resolve_packed_locked resolves them.
static Device::IngressLiterals ingress_literals(zg_engine* e, const char* res_type, const char* relation,
                                               const char* subj_type, const char* subj_rel, const char* one_subj) {
  Device::IngressLiterals lit;
  ResolveMemo memo;
  const zg_rel_str proto{res_type, "", relation, subj_type, one_subj ? one_subj : "", subj_rel};
  resolve_check(e, proto, &lit.base, &memo);
  lit.ok = lit.base.perm != kNone;
  if (lit.ok) {
    lit.rt = memo.parts[memo.last].rt;
    lit.st = memo.parts[memo.last].st;
  }
  if (one_subj) {
    lit.one_subj = one_subj;
    lit.one_len = std::strlen(one_subj);
    lit.one_su = memo.su;
  }
  return lit;
}

extern "C" int zg_resolve_checks_packed_device(zg_engine* e, const char* res_type, const char* relation,
                                               const char* subj_type, const char* subj_rel, const char* d_res_ids,
                                               const uint32_t* d_res_off, const char* d_subj_ids,
                                               const uint32_t* d_subj_off, uint64_t n, zg_check* d_out, void* stream) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!(res_type && relation && subj_type && (n == 0 || (d_res_ids && d_res_off && d_subj_ids && d_out))))
    return fail(ZG_EINVAL, "NULL argument");
  if (int rc = refuse(e, Call::kDeviceBuffers)) return rc;
  if (n == 0) return ZG_OK;
  LOCK_DEVICE(e);
  LOCK_NAMES_SHARED(e);
  const Device::IngressLiterals lit =
      ingress_literals(e, res_type, relation, subj_type, subj_rel, d_subj_off ? nullptr : d_subj_ids);
  std::string err;
  const int rc = e->dev.ingress_resolve(e->store, lit, d_res_ids, d_res_off, d_subj_ids, d_subj_off, n, d_out,
                                        static_cast<cudaStream_t>(stream), &err);
  return rc ? fail(rc, err) : ZG_OK;
}

extern "C" int zg_check_bulk_packed_ingress(zg_engine* e, const char* res_type, const char* relation,
                                            const char* subj_type, const char* subj_rel, const char* res_ids,
                                            const uint32_t* res_off, const char* subj_ids, const uint32_t* subj_off,
                                            uint64_t n, uint8_t* out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!PACKED_ARGS_OK()) return fail(ZG_EINVAL, "NULL argument");
  int rc = refuse(e, Call::kDeviceChecks);
  if (rc) return rc;
  if (n == 0) return ZG_OK;
  rc = publish_if_needed(e);
  if (rc) return rc;
  LOCK_DEVICE(e);
  LOCK_NAMES_SHARED(e);
  const Device::IngressLiterals lit =
      ingress_literals(e, res_type, relation, subj_type, subj_rel, subj_off ? nullptr : subj_ids);
  e->dev.now = now_of(e);
  std::string err;
  rc = e->dev.ingress_check_host(e->store, lit, res_ids, res_off, subj_ids, subj_off, n, out, &err);
  return rc ? fail(rc, err) : ZG_OK;
}

extern "C" int zg_intern_objects_packed(zg_engine* e, int type_id, const char* ids, const uint32_t* off, uint64_t n,
                                        uint32_t* out_ids) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (type_id < 0 || type_id >= static_cast<int>(e->schema.types.size())) return fail(ZG_EINVAL, "unknown type");
  if (n && (!ids || !off || !out_ids)) return fail(ZG_EINVAL, "NULL argument");
  for (uint64_t i = 0; i < n; ++i)
    if (off[i] > off[i + 1]) return fail(ZG_EINVAL, "offsets must not decrease");
  LOCK_NAMES_UNIQUE(e);
  std::string s;
  for (uint64_t i = 0; i < n; ++i) {
    if (off[i] == off[i + 1]) {  // the empty id names no object, as in zg_intern_object
      out_ids[i] = ZG_NO_OBJECT;
      continue;
    }
    s.assign(ids + off[i], off[i + 1] - off[i]);
    out_ids[i] = e->store.intern(type_id, s);
  }
  return ZG_OK;
}

extern "C" int zg_ingress_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const IngressMirror* m = e->dev.ingress_.get();
  out[0] = m ? m->names : 0;
  out[1] = m ? m->device_bytes() : 0;
  out[2] = m ? m->sync_uploads : 0;
  out[3] = m ? m->rebuilds : 0;
  out[4] = m ? m->items_resolved : 0;
  return ZG_OK;
}

// ---- list templates: scanned items -> interned checks without per-item strings --------------

static void utf8_append(uint32_t cp, std::string* out) {
  if (cp < 0x80) {
    out->push_back(static_cast<char>(cp));
  } else if (cp < 0x800) {
    out->push_back(static_cast<char>(0xC0 | (cp >> 6)));
    out->push_back(static_cast<char>(0x80 | (cp & 0x3F)));
  } else if (cp < 0x10000) {
    out->push_back(static_cast<char>(0xE0 | (cp >> 12)));
    out->push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F)));
    out->push_back(static_cast<char>(0x80 | (cp & 0x3F)));
  } else {
    out->push_back(static_cast<char>(0xF0 | (cp >> 18)));
    out->push_back(static_cast<char>(0x80 | ((cp >> 12) & 0x3F)));
    out->push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F)));
    out->push_back(static_cast<char>(0x80 | (cp & 0x3F)));
  }
}

static int hex4(const char* s) {
  int v = 0;
  for (int i = 0; i < 4; ++i) {
    const char h = s[i];
    int d = h >= '0' && h <= '9' ? h - '0' : h >= 'a' && h <= 'f' ? h - 'a' + 10 : h >= 'A' && h <= 'F' ? h - 'A' + 10 : -1;
    if (d < 0) return -1;
    v = v * 16 + d;
  }
  return v;
}

// Appends the decoded contents of a JSON string (the range zg_list_scan recorded, already validated).
static void json_unescape_append(const char* s, size_t n, std::string* out) {
  if (!std::memchr(s, '\\', n)) {
    out->append(s, n);
    return;
  }
  for (size_t i = 0; i < n;) {
    if (s[i] != '\\' || i + 1 >= n) {
      out->push_back(s[i++]);
      continue;
    }
    const char x = s[i + 1];
    i += 2;
    switch (x) {
      case 'b': out->push_back('\b'); break;
      case 'f': out->push_back('\f'); break;
      case 'n': out->push_back('\n'); break;
      case 'r': out->push_back('\r'); break;
      case 't': out->push_back('\t'); break;
      case 'u': {
        int v = i + 4 <= n ? hex4(s + i) : -1;
        if (v < 0) {
          utf8_append(0xFFFD, out);
          break;
        }
        i += 4;
        uint32_t cp = static_cast<uint32_t>(v);
        if (cp >= 0xD800 && cp < 0xDC00 && i + 6 <= n && s[i] == '\\' && s[i + 1] == 'u') {
          const int lo = hex4(s + i + 2);
          if (lo >= 0xDC00 && lo < 0xE000) {
            cp = 0x10000 + ((cp - 0xD800) << 10) + (static_cast<uint32_t>(lo) - 0xDC00);
            i += 6;
          }
        }
        if (cp >= 0xD800 && cp < 0xE000) cp = 0xFFFD;  // lone surrogate, as encoding/json decodes it
        utf8_append(cp, out);
        break;
      }
      default: out->push_back(x);  // \" \\ \/
    }
  }
}

extern "C" int zg_list_resolve(zg_engine* e, const char* body, size_t len, const zg_list_item* items, uint64_t n,
                               const zg_list_template* tpl, zg_check* out, uint8_t* checked) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!tpl || ((!body || !items || !out || !checked) && n)) return fail(ZG_EINVAL, "NULL argument");
  if (tpl->id_kind > ZG_ID_NAMESPACED_NAME) return fail(ZG_EINVAL, "unknown id_kind");
  LOCK_NAMES_SHARED(e);
  // the literal fields once; the resource id per item
  ResolveMemo memo;
  zg_check base;
  const zg_rel_str proto{tpl->res_type, "", tpl->permission, tpl->subj_type, tpl->subj_id, tpl->subj_rel};
  resolve_check(e, proto, &base, &memo);
  const ResolveMemo::SchemaPart& part = memo.parts[memo.last];
  const bool ok = base.perm != kNone;
  const uint32_t su = ok ? memo.su : ZG_NO_OBJECT;
  const std::string req_name = tpl->req_name ? tpl->req_name : "", req_ns = tpl->req_namespace ? tpl->req_namespace : "";
  std::string name, ns, id;
  for (uint64_t i = 0; i < n; ++i) {
    const zg_list_item& it = items[i];
    out[i] = base;
    checked[i] = 0;
    if (!(it.flags & ZG_ITEM_IS_OBJECT)) continue;
    if (it.name_off > len || it.name_len > len - it.name_off || it.ns_off > len || it.ns_len > len - it.ns_off)
      return fail(ZG_EINVAL, "item range outside the body");
    name.clear();
    ns.clear();
    if ((it.flags & ZG_ITEM_HAS_METADATA) && (it.flags & ZG_ITEM_RAW_NAMES)) {
      name.assign(body + it.name_off, it.name_len);
      ns.assign(body + it.ns_off, it.ns_len);
    } else if (it.flags & ZG_ITEM_HAS_METADATA) {
      json_unescape_append(body + it.name_off, it.name_len, &name);
      json_unescape_append(body + it.ns_off, it.ns_len, &ns);
    }
    // pkg/rules/rules.go:312-339
    if (name.empty()) name = req_name;
    if (ns.empty()) ns = req_ns;
    if (tpl->flags & ZG_TPL_CLEAR_NAMESPACE) ns.clear();
    if (tpl->id_kind == ZG_ID_NAMESPACED_NAME && !ns.empty()) {
      id = ns;
      id += '/';
      id += name;
    } else {
      id = name;
    }
    if (id.empty()) continue;  // "T:#perm@..." is not a relationship: the check is skipped
    checked[i] = 1;
    if (!ok) continue;  // unknown type / permission: answers ZG_ITEM_ERROR like the string path
    const uint32_t res = e->store.find(part.rt, id.data(), id.size());
    out[i].res = res;
    uint32_t s2 = su;
    if (s2 == ZG_NO_OBJECT)
      s2 = (res == ZG_NO_OBJECT && part.rt == part.st && tpl->subj_id && id == tpl->subj_id) ? ZG_NO_OBJECT : ZG_NO_OBJECT - 1;
    out[i].subj = s2;
  }
  return ZG_OK;
}

static int list_postfilter_once(zg_engine* e, const char* body, size_t len, const zg_list_template* tpl, uint32_t n_tpl,
                                char* out, size_t cap, size_t* out_len) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!body || !out_len || (!tpl && n_tpl)) return fail(ZG_EINVAL, "NULL argument");
  auto passthrough = [&]() {
    *out_len = len;
    if (len > cap || !out) return static_cast<int>(ZG_E2BIG);
    std::memcpy(out, body, len);
    return static_cast<int>(ZG_OK);
  };
  // one scan in the common case: an item is rarely shorter than 128 bytes (the buffer is not
  // initialised, so its untouched pages cost nothing)
  size_t icap = len / 128 + 16;
  std::unique_ptr<zg_list_item[]> items(new (std::nothrow) zg_list_item[icap]);
  if (!items) return fail(ZG_ENOMEM, "out of host memory");
  uint64_t ib = 0, ie = 0;
  int64_t n = zg_list_scan(body, len, ZG_LIST_ITEMS, items.get(), icap, &ib, &ie);
  if (n == ZG_E2BIG) {
    n = zg_list_scan(body, len, ZG_LIST_ITEMS, nullptr, 0, &ib, &ie);  // count, then one exact rescan
    if (n > 0) {
      icap = static_cast<size_t>(n);
      items.reset(new (std::nothrow) zg_list_item[icap]);
      if (!items) return fail(ZG_ENOMEM, "out of host memory");
      n = zg_list_scan(body, len, ZG_LIST_ITEMS, items.get(), icap, &ib, &ie);
    }
  }
  if (n < 0) return fail(ZG_EINVAL, "failed to parse list response");
  if (n == 0) return passthrough();  // no items array, or an empty one (postfilter.go:25-35)
  const uint64_t N = static_cast<uint64_t>(n);
  std::vector<uint8_t> keep(N, 1), checked(N);
  std::vector<zg_check> one(N), all;
  std::vector<uint64_t> owner;
  for (uint32_t t = 0; t < n_tpl; ++t) {
    int rc = zg_list_resolve(e, body, len, items.get(), N, &tpl[t], one.data(), checked.data());
    if (rc) return rc;
    for (uint64_t i = 0; i < N; ++i)
      if (checked[i]) {
        all.push_back(one[i]);
        owner.push_back(i);
      }
  }
  if (!all.empty()) {
    {
      int rc = publish_if_needed(e);
      if (rc) return rc;
    }
    std::vector<uint8_t> codes(all.size());
    int rc = zg_check_bulk(e, all.data(), all.size(), codes.data());  // ONE launch for the whole list
    if (rc) return rc;
    for (size_t k = 0; k < codes.size(); ++k)
      if (codes[k] != ZG_HAS_PERMISSION) keep[owner[k]] = 0;
  }
  int rc = zg_list_filter(body, len, items.get(), N, keep.data(), ib, ie, ZG_LIST_EMPTY_AS_NULL, out, cap, out_len);
  return rc == ZG_EINVAL ? fail(rc, "zg_list_filter: inconsistent item ranges") : rc;
}

extern "C" int zg_list_postfilter(zg_engine* e, const char* body, size_t len, const zg_list_template* tpl, uint32_t n_tpl,
                                  char* out, size_t cap, size_t* out_len) {
  return with_stable_names(e, [&] { return list_postfilter_once(e, body, len, tpl, n_tpl, out, cap, out_len); });
}

// The steps the handle's LookupResources and LookupSubjects rounds share (run_sharded_lookup, run_sharded_subjects).
// end(dev, err) ends the round on one shard; a failed step ends it on every shard, so that no shard keeps its snapshot
// resident. *waits counts the round's host waits (hl_round_trips / hs_waits), and `what` names the round's buffers in
// out-of-memory messages.
struct HandleRound {
  zg_engine* e;
  int (*end)(Device& dev, std::string* err);
  const char* what;
  uint64_t* waits;
  std::string* err;

  int fail_round(int rc) {
    on_all_devices(e, [&](Device& dev, size_t) { end(dev, nullptr); });
    return rc;
  }
  // fn(device, k, err) on every shard
  template <class F>
  int on_shards(F&& fn) {
    const int rc = on_devices(e, kEveryDevice, fn, err);
    return rc ? fail_round(rc) : ZG_OK;
  }
  // Every shard's candidates as check items in its hl.items, with room for their codes and answer keys: n[k] on shard
  // k. cand(dev, items, cap, &n, err) with items == nullptr asks the capacity items needs. One wait.
  template <class Cand>
  int candidates(Cand&& cand, std::vector<uint64_t>* n) {
    ++*waits;
    return on_shards([&](Device& dev, size_t k, std::string* m) {
      uint64_t need = 0;
      const int rc = cand(dev, nullptr, 0, &need, m);
      if (!rc && (!dev.hl_ensure(dev.hl.items, need * sizeof(zg_check)) || !dev.hl_ensure(dev.hl.codes, need) ||
                  !dev.hl_ensure(dev.hl.routed, need * 8))) {
        *m = std::string("out of device memory (sharded handle ") + what + " candidates)";
        return ZG_ENOMEM;
      }
      return rc ? rc : cand(dev, dev.hl.items.as<zg_check>(), need, &(*n)[k], m);
    });
  }
  // The n[k] checks of every shard's hl.items through the handle's check protocol, where they lie; codes in hl.codes.
  int verify(const std::vector<uint64_t>& n, bool no_wildcards) {
    ShardLists L;
    for (uint32_t k = 0; k < e->n_shards; ++k) {
      L.items.push_back(shard(e, k).hl.items.as<zg_check>());
      L.n.push_back(n[k]);
      L.out.push_back(shard(e, k).hl.codes.as<uint8_t>());
    }
    PeerCounts pc;
    const int rc = run_sharded_lists(e, L, &pc, no_wildcards, err);
    *waits += pc.round_trips;
    return rc ? fail_round(rc) : ZG_OK;
  }
  // The answer keys, gathered on shard 0 (home 0: every key goes there). route(dev, k, counts, err) writes shard k's
  // keys to its hl.routed and counts them by destination; every shard puts them into shard 0's hl.keys behind those of
  // the lower shards. Once every put is done, finish(d0, n_keys, &n_ids, err) sorts and splits them on shard 0 into
  // hl.ids while every other shard ends its round, and the n_ids ids are copied into *host.
  template <class Route, class Finish>
  int gather_keys(Route&& route, Finish&& finish, std::vector<uint32_t>* host) {
    const uint32_t S = e->n_shards;
    std::vector<uint64_t> counts(size_t(S) * S, 0);
    ++*waits;
    if (int rc = on_shards([&](Device& dev, size_t k, std::string* m) { return route(dev, k, &counts[k * S], m); }))
      return rc;
    std::vector<PeerTable> tab(S);
    Device& d0 = e->dev;
    uint64_t n_keys = 0;
    if (!lay_out_inboxes(S, 1, counts, &tab, [&](uint32_t, uint64_t n) -> void* {
          n_keys = n;
          return d0.hl_ensure(d0.hl.keys, n * 8) && d0.hl_ensure(d0.hl.ids, n * 4) ? d0.hl.keys.p : nullptr;
        })) {
      *err = std::string("out of device memory (sharded handle ") + what + " keys)";
      return fail_round(ZG_ENOMEM);
    }
    if (int rc = on_shards([&](Device& dev, size_t k, std::string* m) {
          return dev.peer_put(dev.hl.routed.as<unsigned long long>(), counts[k * S], 1, tab[k], 0, m);
        }))
      return rc;
    std::vector<cudaEvent_t> wait(S);
    for (uint32_t k = 0; k < S; ++k) wait[k] = shard(e, k).peer_event(0);
    uint64_t n_ids = 0;
    ++*waits;
    if (int rc = on_shards([&](Device& dev, size_t k, std::string* m) {
          if (k) return end(dev, m);
          const int wrc = dev.peer_wait(wait, m);
          return wrc ? wrc : finish(dev, n_keys, &n_ids, m);
        }))
      return rc;
    host->resize(n_ids);
    if (n_ids) {
      const cudaError_t ce = cudaSetDevice(d0.device) == cudaSuccess
                                 ? cudaMemcpy(host->data(), d0.hl.ids.p, n_ids * 4, cudaMemcpyDeviceToHost)
                                 : cudaGetLastError();
      ++*waits;
      if (ce != cudaSuccess) {
        *err = std::string("cudaMemcpy (lookup answers): ") + cudaGetErrorString(ce);
        return ZG_ECUDA;
      }
    }
    return ZG_OK;
  }
};

static int end_lookup_round(Device& dev, std::string* err) {
  uint64_t mask = 0, none[kMaxLookupGroup];  // a round holds at most kMaxLookupGroup lookups
  return dev.shard_lookup_finish(nullptr, 0, nullptr, none, &mask, err);
}

static int end_subjects_round(Device& dev, std::string* err) {
  uint64_t listed = 0, excluded = 0;
  return dev.shard_subjects_finish(nullptr, 0, nullptr, &listed, &excluded, err);
}

// LookupResources on a sharded handle (ZG_FLAG_HANDLE_LOOKUPS): one round of dist.DeviceShardedLookup._round over
// reqs[lo, lo + K) (K <= 64), driven in this process; ids[i] / rcs[i] answer reqs[i]. The handle is every rank, so
// every answer goes to shard 0. Shard k owns the objects whose id % S == k and discovers only those in its reverse
// rows, so each object enters the frontier once. Per level, every shard expands the whole replicated frontier (its
// counts and overflow flag: the level's one round trip), then writes its new entries into every shard's next frontier
// behind those of the lower shards (peer_put: the all-gather). The candidates, each on its owner, are verified by the
// handle's check protocol where they lie, and their answer keys gathered on shard 0, sorted and split there.
//
// Why no frontier is overwritten early. (1) A source's new entries (hl.next) are read only by its own peer_put, on
// its own stream, and only its next expand, later on that stream, overwrites them. (2) The put of level L writes
// hl.front[(L + 1) & 1]; the expand of level L reads hl.front[L & 1], and the expand of level L - 1, the last reader of
// hl.front[(L + 1) & 1], has completed on every shard: the host read its counts before it issued any put of level L.
// (3) Every shard's expand of level L + 1 waits on every shard's put event of level L (peer_wait), so it reads the
// whole frontier. The answer keys follow (1) and (3) with shard 0 as the one destination.
static int run_sharded_lookup(zg_engine* e, const std::vector<Device::LookupReq>& reqs, size_t lo, size_t K,
                              std::vector<std::vector<uint32_t>>* ids, std::vector<int>* rcs, std::string* err) {
  const uint32_t S = e->n_shards;
  const std::vector<Device::LookupReq> round(reqs.begin() + static_cast<long>(lo), reqs.begin() + static_cast<long>(lo + K));
  const std::vector<uint8_t> home(K, 0);
  const uint64_t cap = e->dev.lookup_walk_cap();
  HandleRound R{e, end_lookup_round, "lookup", &e->hl_round_trips, err};
  ++e->hl_rounds;
  ++e->hl_round_trips;
  if (int rc = R.on_shards([&](Device& dev, size_t, std::string* m) {
        const int brc = !dev.hl_ensure(dev.hl.front[0], K * 8) || !dev.hl_ensure(dev.hl.next, cap * 8)
                            ? ZG_ENOMEM
                            : dev.shard_lookup_begin(round, home.data(), cap, dev.hl.front[0].as<unsigned long long>(), m);
        if (brc == ZG_ENOMEM && m->empty()) *m = "out of device memory (sharded handle lookup buffers)";
        return brc;
      }))
    return rc;
  // ---- the walk
  const bool exhaustive = !e->dev.use_rbfs;  // ZGPU_NO_RBFS=1: every owned resource of the type is a candidate
  bool overflow = false;
  std::vector<uint64_t> n_out(S);
  std::vector<char> ovf(S);
  std::vector<PeerTable> tab(S);
  std::vector<cudaEvent_t> wait;
  uint64_t n_in = K;
  for (int level = 0; !exhaustive; ++level) {
    ++e->hl_levels;
    ++e->hl_round_trips;
    if (int rc = R.on_shards([&](Device& dev, size_t k, std::string* m) {
          bool o = false;
          int xrc = level ? dev.peer_wait(wait, m) : ZG_OK;
          if (!xrc)
            xrc = dev.shard_lookup_expand(dev.hl.front[level & 1].as<unsigned long long>(), n_in, level,
                                          dev.hl.next.as<unsigned long long>(), &n_out[k], &o, m);
          ovf[k] = o;
          return xrc;
        }))
      return rc;
    uint64_t total = 0;
    for (uint32_t k = 0; k < S; ++k) total += n_out[k];
    overflow = std::find(ovf.begin(), ovf.end(), 1) != ovf.end();
    if (overflow || total == 0 || level == ZG_MAX_DEPTH + 1) break;
    // a gathered frontier past the walk capacity is the overflow the next expand would report on every shard
    if ((overflow = total > cap)) break;
    uint64_t at = 0;
    for (uint32_t k = 0; k < S; ++k) {
      for (uint32_t d = 0; d < S; ++d) tab[k].base[d] = at;
      at += n_out[k];
    }
    for (uint32_t d = 0; d < S; ++d) {
      Device& dev = shard(e, d);
      if (!dev.hl_ensure(dev.hl.front[(level + 1) & 1], total * 8)) {
        *err = "out of device memory (sharded handle lookup frontier)";
        return R.fail_round(ZG_ENOMEM);
      }
      for (uint32_t k = 0; k < S; ++k) tab[k].p[d] = dev.hl.front[(level + 1) & 1].p;
    }
    if (int rc = R.on_shards([&](Device& dev, size_t k, std::string* m) {
          return dev.peer_put(dev.hl.next.as<unsigned long long>(), n_out[k], S, tab[k], level, m);
        }))
      return rc;
    wait.clear();
    for (uint32_t k = 0; k < S; ++k) wait.push_back(shard(e, k).peer_event(level));
    e->hl_frontier += total;
    n_in = total;
  }
  if (overflow && K > 1) {  // checks of the two halves' candidates fit where the whole round's did not
    ++e->hl_halvings;
    const size_t h = K / 2;
    if (int rc = run_sharded_lookup(e, reqs, lo, h, ids, rcs, err)) return rc;
    return run_sharded_lookup(e, reqs, lo + h, K - h, ids, rcs, err);
  }
  const bool every = overflow || exhaustive;
  if (every) ++e->hl_fallbacks;
  // ---- the candidates, verified where they lie
  std::vector<uint64_t> nc(S);
  if (int rc = R.candidates([&](Device& dev, zg_check* items, uint64_t room, uint64_t* n, std::string* m) {
        return dev.shard_lookup_candidates(every, items, room, n, m);
      }, &nc))
    return rc;
  for (uint64_t n : nc) e->hl_candidates += n;
  if (int rc = R.verify(nc, false)) return rc;
  // ---- the answer keys, gathered, sorted and split on shard 0
  std::vector<uint64_t> per(K);
  uint64_t err_mask = 0;
  std::vector<uint32_t> host;
  if (int rc = R.gather_keys(
          [&](Device& dev, size_t k, uint64_t* counts, std::string* m) {
            return dev.shard_lookup_route(dev.hl.codes.as<uint8_t>(), nc[k], S, dev.hl.routed.as<unsigned long long>(),
                                          counts, m);
          },
          [&](Device& d0, uint64_t n_keys, uint64_t* n_ids, std::string* m) {
            const int frc = d0.shard_lookup_finish(d0.hl.keys.as<unsigned long long>(), n_keys, d0.hl.ids.as<uint32_t>(),
                                                   per.data(), &err_mask, m);
            for (uint64_t x : per) *n_ids += x;
            return frc;
          },
          &host))
    return rc;
  uint64_t off = 0;
  for (size_t k = 0; k < K; ++k) {
    if ((err_mask >> k) & 1) (*rcs)[lo + k] = ZG_EDEPTH;
    else (*ids)[lo + k].assign(host.begin() + static_cast<long>(off), host.begin() + static_cast<long>(off + per[k]));
    off += per[k];
  }
  return ZG_OK;
}

// A never-written userset subject T:x#r of a lookup of type T (the subject id is the sentinel): still a member of
// T:x#perm when r is perm itself or a relation inlined into its union. Check decides. Device lock held.
static int never_written_self(zg_engine* e, uint16_t perm, uint16_t stype, uint16_t srel, bool* member, std::string* err) {
  zg_check self{};
  self.res = self.subj = ZG_NO_OBJECT;  // the same never-written object on both sides
  self.perm = perm;
  self.stype = stype;
  self.srel = srel;
  uint8_t code = 0;
  PeerCounts pc;  // a handle checks the one item through its check protocol
  const int rc = is_handle(e) ? run_sharded(e, &self, 1, &code, &pc, err) : e->dev.check_host(&self, 1, &code, err);
  e->hl_round_trips += pc.round_trips;
  if (!rc) *member = code == ZG_HAS_PERMISSION;
  return rc;
}

// Answers a group of queued lookups under the engine lock: cache hits first, the rest in one batched launch
// sequence, then the self-membership of userset subjects (Check is the arbiter of LookupResources).
static void run_lookup_group(zg_engine* e, std::vector<zg_engine::LookupJob*>& group) {  // device lock held
  auto fail_all = [&](int rc, const std::string& msg) {
    for (auto* j : group) {
      j->rc = rc;
      j->err = msg;
    }
  };
  std::string why;
  if (int rc = refuse(e, Call::kLookup, &why)) return fail_all(rc, why);
  const bool handle = is_handle(e);
  if (e->dirty.load() || !e->dev.snap) {  // a handle's failed publish clears every shard's snapshot
    LOCK_NAMES_UNIQUE(e);
    int rc = publish_locked(e);
    if (rc) return fail_all(rc, g_err);
  }
  e->dev.now = now_of(e);
  std::vector<Device::LookupReq> reqs;
  std::vector<size_t> owner;  // job index of each request
  std::vector<int> dup_of(group.size(), -1);
  for (size_t i = 0; i < group.size(); ++i) {
    zg_engine::LookupJob* j = group[i];
    j->key.revision = e->revision;
    j->key.clock = e->clock ? e->clock : -static_cast<int64_t>(e->dev.now);  // wall clock: valid within the same second
    bool hit = false;
    for (const auto& c : e->lookup_cache)
      if (c.first == j->key) {
        j->ids = *c.second;
        hit = true;
        break;
      }
    if (hit) continue;
    for (size_t k = 0; k < i && dup_of[i] < 0; ++k)
      if (group[k]->key == j->key && dup_of[k] < 0) dup_of[i] = static_cast<int>(k);
    if (dup_of[i] >= 0) continue;
    zg_check proto{};
    proto.subj = j->key.subj;
    proto.perm = j->key.perm;
    proto.stype = j->key.stype;
    proto.srel = j->key.srel;
    reqs.push_back(Device::LookupReq{j->key.res_type, proto});
    owner.push_back(i);
  }
  if (!reqs.empty()) {
    std::vector<std::vector<uint32_t>> ids;
    std::vector<int> rcs;
    std::string err;
    int rc = ZG_OK;
    const size_t nd = 1 + e->replicas.size();
    if (handle) {
      ids.resize(reqs.size());
      rcs.assign(reqs.size(), ZG_OK);
      rc = run_sharded_lookup(e, reqs, 0, reqs.size(), &ids, &rcs, &err);
      if (reqs.size() > 1) {
        ++e->dev.lookup_batches;
        e->dev.lookups_batched += reqs.size();
      }
    } else if (nd == 1 || reqs.size() < 2) {
      rc = e->dev.lookup_batch(reqs, &ids, &rcs, &err);
    } else {
      // replicas: the lookups of the group are dealt out to the devices
      std::vector<std::vector<Device::LookupReq>> part(nd);
      std::vector<std::vector<size_t>> which(nd);
      for (size_t r = 0; r < reqs.size(); ++r) {
        part[r % nd].push_back(reqs[r]);
        which[r % nd].push_back(r);
      }
      std::vector<std::vector<std::vector<uint32_t>>> pids(nd);
      std::vector<std::vector<int>> prcs(nd);
      const uint32_t now = e->dev.now;
      rc = on_devices(e, kEveryDevice, [&](Device& dev, size_t i, std::string* m) {
        dev.now = now;
        return part[i].empty() ? ZG_OK : dev.lookup_batch(part[i], &pids[i], &prcs[i], m);
      }, &err);
      ids.resize(reqs.size());
      rcs.assign(reqs.size(), ZG_OK);
      for (size_t i = 0; i < nd && !rc; ++i)
        for (size_t k = 0; k < which[i].size(); ++k) {
          ids[which[i][k]] = std::move(pids[i][k]);
          rcs[which[i][k]] = prcs[i][k];
        }
    }
    if (rc) return fail_all(rc, err);
    for (size_t r = 0; r < reqs.size(); ++r) {
      zg_engine::LookupJob* j = group[owner[r]];
      if (rcs[r]) {
        j->rc = rcs[r];
        j->err = "LookupResources: a candidate could not be decided (max dispatch depth / work budget exceeded)";
        continue;
      }
      j->ids = std::move(ids[r]);
      // A userset subject T:x#r is a member of T:x#P for every relation r inlined into P's union, with or
      // without relationships, and the reverse walk only reaches x through stored edges: ask the check
      // kernel about the one candidate res = subj. (A handle's round made it a candidate on x's owner.)
      const zg_engine::LookupKey& k = j->key;
      if (!handle && k.srel != kNone && k.stype == k.res_type && k.subj < ZG_NO_OBJECT - 1 &&
          !std::binary_search(j->ids.begin(), j->ids.end(), k.subj)) {
        zg_check self = reqs[r].proto;
        self.res = k.subj;
        uint8_t code = 0;
        rc = e->dev.check_host(&self, 1, &code, &err);
        if (rc) {
          j->rc = rc;
          j->err = err;
          continue;
        }
        if (code == ZG_HAS_PERMISSION) j->ids.insert(std::upper_bound(j->ids.begin(), j->ids.end(), k.subj), k.subj);
      }
      e->lookup_cache.emplace_back(k, std::make_shared<const std::vector<uint32_t>>(j->ids));
      while (e->lookup_cache.size() > zg_engine::kLookupCache) e->lookup_cache.pop_front();
    }
  }
  for (size_t i = 0; i < group.size(); ++i) {
    zg_engine::LookupJob* j = group[i];
    if (dup_of[i] >= 0) {
      const zg_engine::LookupJob* src = group[dup_of[i]];
      j->ids = src->ids;
      j->rc = src->rc;
      j->err = src->err;
    }
    if (!j->rc && j->want_self && j->key.srel != kNone && j->key.stype == j->key.res_type && j->key.subj >= ZG_NO_OBJECT - 1) {
      std::string cerr;
      if (int crc = never_written_self(e, j->key.perm, j->key.stype, j->key.srel, &j->self_member, &cerr)) {
        j->rc = crc;
        j->err = cerr;
      }
    }
  }
}

// Queue one lookup; the first caller to arrive while nobody leads answers everything queued (<= 64 per
// launch sequence). Must be called WITHOUT e->mu held.
static int lookup_queued(zg_engine* e, uint16_t res_type, uint16_t perm, uint16_t stype, uint32_t subj, uint16_t srel,
                         std::vector<uint32_t>* ids, bool* self_member = nullptr) {
  if (self_member) *self_member = false;
  const Schema& sc = e->schema;
  if (res_type >= sc.types.size() || perm >= sc.slots.size() || sc.slots[perm].type != res_type)
    return fail(ZG_EINVAL, "unknown resource type or permission");
  if (stype >= sc.types.size() || (srel != kNone && (srel >= sc.slots.size() || sc.slots[srel].type != stype)))
    return fail(ZG_EINVAL, "unknown subject type or relation");
  zg_engine::LookupJob me;
  me.key.subj = subj;
  me.key.res_type = res_type;
  me.key.perm = perm;
  me.key.stype = stype;
  me.key.srel = srel;
  me.want_self = self_member != nullptr;
  e->lookups.submit(
      &me, e->mu,
      [](const std::vector<zg_engine::LookupJob*>& queue) { return std::min<size_t>(queue.size(), kMaxLookupGroup); },
      [e](std::vector<zg_engine::LookupJob*>& group) { run_lookup_group(e, group); });
  if (me.rc) return fail(me.rc, me.err);
  *ids = std::move(me.ids);
  if (self_member) *self_member = me.self_member;
  return ZG_OK;
}

extern "C" int zg_lookup_resources(zg_engine* e, uint16_t res_type, uint16_t perm, uint16_t stype, uint32_t subj,
                                   uint16_t srel, uint32_t* out_ids, uint64_t cap, uint64_t* n_out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!n_out) return fail(ZG_EINVAL, "NULL n_out");
  // no lock here: the call QUEUES behind a running group (the group's leader validates the engine state)
  std::vector<uint32_t> ids;
  int rc = lookup_queued(e, res_type, perm, stype, subj, srel, &ids);
  if (rc) return rc;
  *n_out = ids.size();
  if (ids.size() > cap || (!out_ids && !ids.empty())) return ZG_E2BIG;
  if (!ids.empty()) std::memcpy(out_ids, ids.data(), ids.size() * 4);
  return ZG_OK;
}

// (resource type, permission, subject) strings -> ids, under the engine lock. su == ZG_NO_OBJECT: never written.
static int resolve_lookup_strs(zg_engine* e, const char* res_type, const char* perm, const char* subj_type, const char* subj_id,
                               const char* subj_rel, int* rt, int* p, int* st, uint16_t* sr, uint32_t* su) {
  int rc = publish_if_needed(e);
  if (rc) return rc;
  LOCK_NAMES_SHARED(e);
  const Schema& sc = e->schema;
  *rt = sc.type_id(res_type);
  *st = sc.type_id(subj_type);
  if (*rt < 0) return fail(ZG_EINVAL, std::string("object definition `") + res_type + "` not found");
  if (*st < 0) return fail(ZG_EINVAL, std::string("object definition `") + subj_type + "` not found");
  *p = sc.slot_id(*rt, perm);
  if (*p < 0) return fail(ZG_EINVAL, std::string("relation/permission `") + perm + "` not found under definition `" + res_type + "`");
  *sr = kNone;
  if (!none_rel(subj_rel)) {
    int s = sc.slot_id(*st, subj_rel);
    if (s < 0) return fail(ZG_EINVAL, std::string("relation `") + subj_rel + "` not found under definition `" + subj_type + "`");
    *sr = static_cast<uint16_t>(s);
  }
  *su = e->store.find(*st, subj_id);
  return ZG_OK;
}

static int lookup_resources_str_once(zg_engine* e, const char* res_type, const char* perm, const char* subj_type,
                                     const char* subj_id, const char* subj_rel, char* buf, size_t cap, size_t* need,
                                     uint64_t* n_out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!res_type || !perm || !subj_type || !subj_id) return fail(ZG_EINVAL, "NULL argument");
  int rt, p, st;
  uint16_t sr;
  uint32_t su;
  int rc = resolve_lookup_strs(e, res_type, perm, subj_type, subj_id, subj_rel, &rt, &p, &st, &sr, &su);
  if (rc) return rc;
  std::vector<uint32_t> ids;
  bool self_member = false;
  rc = lookup_queued(e, static_cast<uint16_t>(rt), static_cast<uint16_t>(p), static_cast<uint16_t>(st),
                     su == ZG_NO_OBJECT ? ZG_NO_OBJECT - 1 : su, sr, &ids, &self_member);
  if (rc) return rc;
  if (e->resolve_hook) e->resolve_hook(e->resolve_hook_arg);
  std::vector<std::string> names;
  {
    LOCK_NAMES_SHARED(e);
    for (uint32_t id : ids) {
      std::string_view n;
      names.push_back(e->store.name(rt, id, &n) ? std::string(n) : std::to_string(id));
    }
  }
  // never-written userset subject that names itself
  if (su == ZG_NO_OBJECT && self_member) names.push_back(subj_id);
  size_t total = 1;
  for (const auto& n : names) total += n.size() + 1;
  if (need) *need = total;
  if (n_out) *n_out = names.size();
  if (total > cap || !buf) return ZG_E2BIG;
  size_t w = 0;
  for (const auto& n : names) {
    std::memcpy(buf + w, n.data(), n.size());
    w += n.size();
    buf[w++] = '\n';
  }
  buf[w] = 0;
  return ZG_OK;
}

extern "C" int zg_lookup_resources_str(zg_engine* e, const char* res_type, const char* perm, const char* subj_type,
                                       const char* subj_id, const char* subj_rel, char* buf, size_t cap, size_t* need,
                                       uint64_t* n_out) {
  return with_stable_names(e, [&] {
    return lookup_resources_str_once(e, res_type, perm, subj_type, subj_id, subj_rel, buf, cap, need, n_out);
  });
}

// ---- pages of LookupResources: zg_lookup_resources_page, zg_lookup_resources_page_str ----

// The request a lookup cursor was made for: the resolved type, permission, subject type and subject relation ids, the
// form, and the subject as given (its id in the id form, its name in the string form: a name need not exist).
static uint64_t lookup_fingerprint(uint16_t rt, uint16_t perm, uint16_t st, uint16_t srel, const char* subj_name,
                                   uint32_t subj) {
  uint64_t h = 0xcbf29ce484222325ull;
  auto mix = [&](const void* p, size_t n) {
    for (size_t i = 0; i < n; ++i) h = (h ^ static_cast<const uint8_t*>(p)[i]) * 0x100000001b3ull;
  };
  mix("LookupResources", 15);
  const uint16_t ids[5] = {rt, perm, st, srel, static_cast<uint16_t>(subj_name ? 1 : 0)};
  mix(ids, sizeof ids);
  if (subj_name) {
    const size_t n = std::strlen(subj_name);
    mix(&n, sizeof n);
    mix(subj_name, n);
  } else {
    mix(&subj, sizeof subj);
  }
  return h;
}

// *after -> *c (zeroed when after is NULL: the start). ZG_EINVAL for a read cursor, a cursor of another request or
// form, or one made before the schema was loaded again.
static int lookup_cursor(const zg_engine* e, const zg_read_cursor* after, uint64_t fp, bool str_form, CursorBits* c) {
  *c = CursorBits{};
  if (!after) return ZG_OK;
  std::memcpy(c, after->opaque, sizeof *c);
  if (c->version != kLookupCursorVersion || c->has_key > (str_form ? kPastIds : 1))
    return fail(ZG_EINVAL, "lookup cursor: not a LookupResources cursor of this engine");
  if (c->schema_gen != e->schema_gen || c->fp != fp)
    return fail(ZG_EINVAL, "lookup cursor: it was made for another lookup or under another schema");
  return ZG_OK;
}

static zg_read_cursor lookup_cursor_at(const zg_engine* e, uint64_t fp, uint16_t rt, uint32_t id, uint16_t has_key = 1) {
  const PageKey k{rt, id, 0, 0};
  return make_cursor(e, fp, &k, kLookupCursorVersion, has_key);
}

// One page of LookupResources: the first `limit` ids of the unpaged answer after `after` (every id when !has_after) in
// *ids, *more = 1 when another id follows. A replicated engine verifies windows of the candidates on its first device
// (Device::lookup_page); a sharded handle runs its whole round and cuts the page from the answer. self_member (NULL:
// not asked): whether the never-written userset subject is a member of itself, asked only once the ids ran out.
static int lookup_page_ids(zg_engine* e, uint16_t rt, uint16_t perm, uint16_t st, uint32_t subj, uint16_t srel, uint64_t limit,
                           bool has_after, uint32_t after, std::vector<uint32_t>* ids, bool* more, bool* self_member) {
  if (int rc = refuse(e, Call::kLookup)) return rc;
  LOCK_DEVICE(e);
  if (e->dirty.load() || !e->dev.snap) {  // a handle's failed publish clears every shard's snapshot
    LOCK_NAMES_UNIQUE(e);
    if (int rc = publish_locked(e)) return rc;
  }
  const uint32_t now = now_of(e);
  const uint64_t want = std::min<uint64_t>(limit, ZG_NO_OBJECT) + 1;  // no type holds more ids than that
  zg_check proto{};
  proto.subj = subj;
  proto.perm = perm;
  proto.stype = st;
  proto.srel = srel;
  std::string err;
  if (is_handle(e)) {
    for (uint32_t k = 0; k < e->n_shards; ++k) shard(e, k).now = now;
    std::vector<std::vector<uint32_t>> all(1);
    std::vector<int> rcs(1, ZG_OK);
    if (int rc = run_sharded_lookup(e, {Device::LookupReq{rt, proto}}, 0, 1, &all, &rcs, &err)) return fail(rc, err);
    if (rcs[0])  // the round reports an undecidable candidate per lookup, not per id: the page fails as the whole call
      return fail(rcs[0], "LookupResources: a candidate could not be decided (max dispatch depth / work budget exceeded)");
    const auto from = has_after ? std::upper_bound(all[0].begin(), all[0].end(), after) : all[0].begin();
    const uint64_t left = static_cast<uint64_t>(all[0].end() - from);
    ids->assign(from, from + static_cast<long>(std::min(left, want)));
    ++e->lp_cut;
    e->lp_after += left;
  } else {
    // the userset subject's own object is a candidate (the walk reaches it only through stored edges)
    const uint32_t self = srel != kNone && st == rt && subj < ZG_NO_OBJECT - 1 ? subj : ZG_NO_OBJECT;
    Device::LookupPageStats ps;
    e->dev.now = now;
    if (int rc = e->dev.lookup_page(rt, proto, has_after, after, want, self, ids, &ps, &err)) return fail(rc, err);
    ++e->lp_windowed;
    e->lp_after += ps.after;
    e->lp_verified += ps.verified;
    e->lp_windows += ps.windows;
  }
  *more = ids->size() > limit;
  if (*more) ids->resize(limit);
  if (self_member) {
    *self_member = false;
    if (!*more && srel != kNone && st == rt) {
      if (int rc = never_written_self(e, perm, st, srel, self_member, &err)) return fail(rc, err);
    }
  }
  return ZG_OK;
}

extern "C" int zg_lookup_resources_page(zg_engine* e, uint16_t res_type, uint16_t perm, uint16_t stype, uint32_t subj,
                                        uint16_t srel, uint64_t limit, const zg_read_cursor* after, uint32_t* ids,
                                        uint64_t* n_out, zg_read_cursor* cursors, zg_read_cursor* next, int32_t* more) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!ids || !n_out) return fail(ZG_EINVAL, "NULL ids / n_out");
  if (limit == 0) return fail(ZG_EINVAL, "page limit must be at least 1 (zg_lookup_resources looks up without one)");
  const Schema& sc = e->schema;
  if (res_type >= sc.types.size() || perm >= sc.slots.size() || sc.slots[perm].type != res_type)
    return fail(ZG_EINVAL, "unknown resource type or permission");
  if (stype >= sc.types.size() || (srel != kNone && (srel >= sc.slots.size() || sc.slots[srel].type != stype)))
    return fail(ZG_EINVAL, "unknown subject type or relation");
  const uint64_t fp = lookup_fingerprint(res_type, perm, stype, srel, nullptr, subj);
  CursorBits c;
  if (int rc = lookup_cursor(e, after, fp, false, &c)) return rc;
  std::vector<uint32_t> got;
  bool has_more = false;
  if (int rc = lookup_page_ids(e, res_type, perm, stype, subj, srel, limit, c.has_key, c.key.res, &got, &has_more, nullptr))
    return rc;
  *n_out = got.size();
  if (!got.empty()) std::memcpy(ids, got.data(), got.size() * 4);
  if (cursors)
    for (size_t i = 0; i < got.size(); ++i) cursors[i] = lookup_cursor_at(e, fp, res_type, got[i]);
  if (next) *next = got.empty() ? (after ? *after : make_cursor(e, fp, nullptr, kLookupCursorVersion))
                                : lookup_cursor_at(e, fp, res_type, got.back());
  if (more) *more = has_more;
  return ZG_OK;
}

static int lookup_page_str_once(zg_engine* e, const char* res_type, const char* perm, const char* subj_type,
                                const char* subj_id, const char* subj_rel, uint64_t limit, const zg_read_cursor* after,
                                char* buf, size_t cap, size_t* need, uint64_t* n_out, zg_read_cursor* cursors,
                                zg_read_cursor* next, int32_t* more) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!res_type || !perm || !subj_type || !subj_id) return fail(ZG_EINVAL, "NULL argument");
  if (limit == 0) return fail(ZG_EINVAL, "page limit must be at least 1 (zg_lookup_resources_str looks up without one)");
  int rt, p, st;
  uint16_t sr;
  uint32_t su;
  if (int rc = resolve_lookup_strs(e, res_type, perm, subj_type, subj_id, subj_rel, &rt, &p, &st, &sr, &su)) return rc;
  const uint64_t fp = lookup_fingerprint(static_cast<uint16_t>(rt), static_cast<uint16_t>(p), static_cast<uint16_t>(st), sr,
                                         subj_id, 0);
  CursorBits c;
  if (int rc = lookup_cursor(e, after, fp, true, &c)) return rc;
  std::vector<uint32_t> ids;
  bool has_more = false, self_member = false;
  if (c.has_key != kPastIds) {  // past the ids, the never-written subject's own name was the last line
    const bool never_written = su == ZG_NO_OBJECT;
    if (int rc = lookup_page_ids(e, static_cast<uint16_t>(rt), static_cast<uint16_t>(p), static_cast<uint16_t>(st),
                                 never_written ? ZG_NO_OBJECT - 1 : su, sr, limit, c.has_key, c.key.res, &ids, &has_more,
                                 never_written ? &self_member : nullptr))
      return rc;
  } else if (int rc = refuse(e, Call::kLookup)) {
    return rc;
  }
  if (e->resolve_hook) e->resolve_hook(e->resolve_hook_arg);
  // the never-written subject that names itself comes after every id
  const bool self_line = self_member && ids.size() < limit;
  if (self_member && !self_line) has_more = true;
  std::vector<std::string> names;
  {
    LOCK_NAMES_SHARED(e);
    for (uint32_t id : ids) {
      std::string_view n;
      names.push_back(e->store.name(rt, id, &n) ? std::string(n) : std::to_string(id));
    }
  }
  if (self_line) names.push_back(subj_id);
  size_t total = 1;
  for (const auto& n : names) total += n.size() + 1;
  if (need) *need = total;
  if (n_out) *n_out = names.size();
  if (total > cap || !buf) return ZG_E2BIG;
  size_t w = 0;
  for (const auto& n : names) {
    std::memcpy(buf + w, n.data(), n.size());
    w += n.size();
    buf[w++] = '\n';
  }
  buf[w] = 0;
  const uint16_t t = static_cast<uint16_t>(rt);
  if (cursors) {
    for (size_t i = 0; i < ids.size(); ++i) cursors[i] = lookup_cursor_at(e, fp, t, ids[i]);
    if (self_line) cursors[ids.size()] = lookup_cursor_at(e, fp, t, 0, kPastIds);
  }
  if (next) {
    if (self_line) *next = lookup_cursor_at(e, fp, t, 0, kPastIds);
    else if (!ids.empty()) *next = lookup_cursor_at(e, fp, t, ids.back());
    else *next = after ? *after : make_cursor(e, fp, nullptr, kLookupCursorVersion);
  }
  if (more) *more = has_more;
  return ZG_OK;
}

extern "C" int zg_lookup_resources_page_str(zg_engine* e, const char* res_type, const char* perm, const char* subj_type,
                                            const char* subj_id, const char* subj_rel, uint64_t limit,
                                            const zg_read_cursor* after, char* buf, size_t cap, size_t* need,
                                            uint64_t* n_out, zg_read_cursor* cursors, zg_read_cursor* next, int32_t* more) {
  return with_stable_names(e, [&] {
    return lookup_page_str_once(e, res_type, perm, subj_type, subj_id, subj_rel, limit, after, buf, cap, need, n_out,
                                cursors, next, more);
  });
}

extern "C" int zg_lookup_page_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  const uint64_t c[5] = {e->lp_windowed.load(), e->lp_cut.load(), e->lp_after.load(), e->lp_verified.load(),
                         e->lp_windows.load()};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

// ---- LookupSubjects --------------------------------------------------------------------------

// LookupSubjects on a sharded handle (ZG_FLAG_HANDLE_SUBJECTS): one round of dist.DeviceShardedLookup's
// _subjects_round with one lookup (home 0), driven in this process; every call runs its own round on every shard.
// Shard k holds the forward rows of the objects it owns, but the subjects in them can be owned by any shard, so each
// discovery goes to its owner, which admits it once per lookup (the owner of req.res seeds the walk and holds the
// probe). Per level, every shard expands its own frontier into its outbox and counts the outbox by owner on the device;
// the host reads every shard's overflow flag and counts (the level's first wait), lays out every owner's inbox from
// them, and every shard writes its outbox straight into the owners' inboxes (peer memory). Each owner admits what
// arrived once every shard's scatter of the level is done (events); its admitted count sizes its next expand (the
// second wait). Levels 0 .. ZG_MAX_DEPTH + 1 are expanded, as on a replica, and one more count reports the last
// admissions' overflow. An overflow goes straight to the exhaustive candidates: a single lookup is not halved. The
// candidates are verified where they lie by the handle's check protocol; the probe verdicts of the shards are OR-ed
// on the host (the handle is every rank); when the wildcard is granted, the HAS candidates are verified again with
// no wildcard relationship visible on any pass of any shard; the answer keys are gathered, sorted and split on shard 0.
//
// Why no buffer is overwritten before it is read. (1) A shard's outbox is read only by its own scatter, on its own
// stream, and only its next expand, later on that stream, overwrites it. (2) Shard d's inbox (hl.inbox) is written by
// every shard's scatter of level L and read by d's admit of level L, which waits on every shard's scatter event of
// level L (peer_wait). No scatter of level L + 1 is issued before the host has waited for every admit of level L (the
// admitted counts), so one inbox per shard is enough; the inbox is grown only while every shard is idle. (3) A shard's
// frontier (hl.front[0]) is read by its expand and rewritten by its admit, in that order on its stream. The answer
// keys follow (1) and (2) with shard 0 as the one destination. The walk buffers and hl are shared with the handle's
// LookupResources round (run_sharded_lookup); both run under the device lock, so they never interleave.
static int run_sharded_subjects(zg_engine* e, const Device::SubjectsReq& req, bool include, Device::SubjectsAnswer* ans,
                                std::string* err) {
  *ans = Device::SubjectsAnswer{};
  const uint32_t S = e->n_shards;
  const std::vector<Device::SubjectsReq> round{req};
  const uint8_t home = 0;
  const uint64_t cap = e->dev.lookup_walk_cap();
  HandleRound R{e, end_subjects_round, "subjects", &e->hs_waits, err};
  ++e->hs_lookups;
  std::vector<uint64_t> n_front(S, 0);
  ++e->hs_waits;
  if (int rc = R.on_shards([&](Device& dev, size_t k, std::string* m) {
        const int brc = !dev.hl_ensure(dev.hl.front[0], cap * 8)
                            ? ZG_ENOMEM
                            : dev.shard_subjects_begin(round, &home, include ? 1 : 0, cap,
                                                       dev.hl.front[0].as<unsigned long long>(), &n_front[k], m);
        if (brc == ZG_ENOMEM && m->empty()) *m = "out of device memory (sharded handle subjects frontier)";
        return brc;
      }))
    return rc;
  // ---- the walk
  const bool exhaustive = !e->dev.use_rbfs;  // ZGPU_NO_RBFS=1: every owned object of the subject type is a candidate
  bool overflow = false;
  std::vector<uint64_t> counts(size_t(S) * S, 0), arrived(S, 0);
  std::vector<char> ovf(S);
  std::vector<PeerTable> tab(S);
  std::vector<cudaEvent_t> wait(S);
  for (int level = 0; !exhaustive; ++level) {
    const bool expand = level <= ZG_MAX_DEPTH + 1;
    ++e->hs_waits;
    if (int rc = R.on_shards([&](Device& dev, size_t k, std::string* m) {
          bool o = false;
          const int xrc = dev.shard_subjects_expand_count(dev.hl.front[0].as<unsigned long long>(), expand ? n_front[k] : 0,
                                                          &counts[k * S], &o, m);
          ovf[k] = o;
          return xrc;
        }))
      return rc;
    if ((overflow = std::find(ovf.begin(), ovf.end(), 1) != ovf.end())) break;
    if (!expand || std::all_of(n_front.begin(), n_front.end(), [](uint64_t n) { return n == 0; })) break;
    ++e->hs_levels;
    if (!lay_out_inboxes(S, S, counts, &tab, [&](uint32_t d, uint64_t n) -> void* {
          for (uint32_t k = 0; k < S; ++k)
            if (k != d) e->hs_entries += counts[size_t(k) * S + d];
          arrived[d] = n;
          Device& dev = shard(e, d);
          return dev.hl_ensure(dev.hl.inbox, n * 8) ? dev.hl.inbox.p : nullptr;
        })) {
      *err = "out of device memory (sharded handle subjects inbox)";
      return R.fail_round(ZG_ENOMEM);
    }
    if (int rc = R.on_shards([&](Device& dev, size_t k, std::string* m) {
          uint64_t n = 0;
          for (uint32_t d = 0; d < S; ++d) n += counts[k * S + d];
          return dev.shard_subjects_scatter(n, tab[k], level, m);
        }))
      return rc;
    for (uint32_t k = 0; k < S; ++k) wait[k] = shard(e, k).peer_event(level);
    ++e->hs_waits;
    if (int rc = R.on_shards([&](Device& dev, size_t k, std::string* m) {
          const int wrc = dev.peer_wait(wait, m);
          return wrc ? wrc
                     : dev.shard_subjects_admit(dev.hl.inbox.as<unsigned long long>(), arrived[k],
                                                dev.hl.front[0].as<unsigned long long>(), &n_front[k], m);
        }))
      return rc;
  }
  const bool every = overflow || exhaustive;
  if (every) ++e->hs_fallbacks;
  // ---- the first verification, where the candidates lie
  std::vector<uint64_t> nc(S, 0);
  if (int rc = R.candidates([&](Device& dev, zg_check* items, uint64_t room, uint64_t* n, std::string* m) {
        return dev.shard_subjects_candidates(every, items, room, n, m);
      }, &nc))
    return rc;
  for (uint64_t n : nc) {
    e->hs_candidates += n;
    ans->n_verified += n;
  }
  if (int rc = R.verify(nc, false)) return rc;
  std::vector<uint64_t> granted(S, 0), failed(S, 0);
  ++e->hs_waits;
  if (int rc = R.on_shards([&](Device& dev, size_t k, std::string* m) {
        return dev.shard_subjects_verdicts(dev.hl.codes.as<uint8_t>(), nc[k], &granted[k], &failed[k], m);
      }))
    return rc;
  uint64_t g = 0, f = 0;  // the probe's verdict is on the resource's owner, a failed candidate anywhere
  for (uint32_t k = 0; k < S; ++k) {
    g |= granted[k];
    f |= failed[k];
  }
  if (f & 1) {
    *err = "LookupSubjects: a subject could not be decided (max dispatch depth / work budget exceeded)";
    return R.fail_round(ZG_EDEPTH);
  }
  // ---- the keys of the first verification, and the no-wildcards verification of the HAS candidates when granted.
  // Its items and codes take the place of the first verification's, which shard_subjects_nowild has read (it waits).
  std::vector<uint64_t> nnw(S, 0);
  ++e->hs_waits;
  if (int rc = R.on_shards([&](Device& dev, size_t k, std::string* m) {
        return dev.shard_subjects_nowild(dev.hl.codes.as<uint8_t>(), nc[k], g, f, dev.hl.items.as<zg_check>(), nc[k],
                                         &nnw[k], m);
      }))
    return rc;
  if (g & 1) {
    for (uint64_t n : nnw) e->hs_nowild += n;
    if (int rc = R.verify(nnw, true)) return rc;
  }
  // ---- the answer keys, gathered, sorted and split on shard 0
  uint64_t listed = 0, excluded = 0;
  std::vector<uint32_t> host;
  if (int rc = R.gather_keys(
          [&](Device& dev, size_t k, uint64_t* to, std::string* m) {
            return dev.shard_subjects_route(dev.hl.codes.as<uint8_t>(), nnw[k], S, dev.hl.routed.as<unsigned long long>(),
                                            to, m);
          },
          [&](Device& d0, uint64_t n_keys, uint64_t* n_ids, std::string* m) {
            const int frc = d0.shard_subjects_finish(d0.hl.keys.as<unsigned long long>(), n_keys, d0.hl.ids.as<uint32_t>(),
                                                     &listed, &excluded, m);
            *n_ids = listed + excluded;
            return frc;
          },
          &host))
    return rc;
  ans->ids.assign(host.begin(), host.begin() + static_cast<long>(listed));
  ans->wildcard = (g & 1) && include;
  if (ans->wildcard) ans->excluded.assign(host.begin() + static_cast<long>(listed), host.end());
  ans->fell_back = every;
  return ZG_OK;
}

// Arguments are checked before anything else (a host-only engine still reports ZG_EINVAL for them). The
// device lock is FIFO, as for a single LookupResources; a multi-device engine answers on its first device, a sharded
// handle with ZG_FLAG_HANDLE_SUBJECTS on every shard (run_sharded_subjects).
static int lookup_subjects_ids(zg_engine* e, uint16_t perm, uint32_t res, uint16_t stype, uint16_t srel, uint32_t option,
                               Device::SubjectsAnswer* ans) {
  const Schema& sc = e->schema;
  if (perm >= sc.slots.size()) return fail(ZG_EINVAL, "unknown permission");
  if (stype >= sc.types.size() || (srel != kNone && (srel >= sc.slots.size() || sc.slots[srel].type != stype)))
    return fail(ZG_EINVAL, "unknown subject type or relation");
  if (option != ZG_WILDCARDS_INCLUDE && option != ZG_WILDCARDS_EXCLUDE) return fail(ZG_EINVAL, "unknown wildcard option");
  if (int rc = refuse(e, Call::kSubjects)) return rc;
  LOCK_DEVICE(e);
  if (e->dirty.load() || !e->dev.snap) {  // a handle's failed publish clears every shard's snapshot
    LOCK_NAMES_UNIQUE(e);
    int rc = publish_locked(e);
    if (rc) return rc;
  }
  const uint32_t now = now_of(e);
  std::string err;
  int rc = ZG_OK;
  if (serves_subjects(e)) {
    for (uint32_t k = 0; k < e->n_shards; ++k) shard(e, k).now = now;
    const Device::SubjectsReq req{res, static_cast<uint16_t>(sc.slots[perm].type), perm, stype, srel};
    rc = run_sharded_subjects(e, req, option == ZG_WILDCARDS_INCLUDE, ans, &err);
  } else {
    e->dev.now = now;
    rc = e->dev.lookup_subjects(sc.slots[perm].type, res, perm, stype, srel, option == ZG_WILDCARDS_INCLUDE, ans, &err);
  }
  return rc ? fail(rc, err) : ZG_OK;
}

extern "C" int zg_lookup_subjects(zg_engine* e, uint16_t perm, uint32_t res, uint16_t stype, uint16_t srel,
                                  uint32_t wildcard_option, uint32_t* ids, uint64_t cap, uint64_t* n_out, uint32_t* excluded,
                                  uint64_t ex_cap, uint64_t* n_excluded, int32_t* wildcard) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!n_out || !n_excluded || !wildcard) return fail(ZG_EINVAL, "NULL n_out / n_excluded / wildcard");
  Device::SubjectsAnswer ans;
  int rc = lookup_subjects_ids(e, perm, res, stype, srel, wildcard_option, &ans);
  if (rc) return rc;
  *n_out = ans.ids.size();
  *n_excluded = ans.excluded.size();
  *wildcard = ans.wildcard ? 1 : 0;
  if (ans.ids.size() > cap || ans.excluded.size() > ex_cap || (!ids && !ans.ids.empty()) ||
      (!excluded && !ans.excluded.empty()))
    return ZG_E2BIG;
  if (!ans.ids.empty()) std::memcpy(ids, ans.ids.data(), ans.ids.size() * 4);
  if (!ans.excluded.empty()) std::memcpy(excluded, ans.excluded.data(), ans.excluded.size() * 4);
  return ZG_OK;
}

static int lookup_subjects_str_once(zg_engine* e, const char* res_type, const char* res_id, const char* perm,
                                    const char* subj_type, const char* subj_rel, uint32_t wildcard_option, char* buf,
                                    size_t cap, size_t* need, uint64_t* n_out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!res_type || !res_id || !perm || !subj_type) return fail(ZG_EINVAL, "NULL argument");
  int rt, p, st;
  uint16_t sr = kNone;
  uint32_t res;
  {
    LOCK_NAMES_SHARED(e);
    const Schema& sc = e->schema;
    rt = sc.type_id(res_type);
    st = sc.type_id(subj_type);
    if (rt < 0) return fail(ZG_EINVAL, std::string("object definition `") + res_type + "` not found");
    if (st < 0) return fail(ZG_EINVAL, std::string("object definition `") + subj_type + "` not found");
    p = sc.slot_id(rt, perm);
    if (p < 0) return fail(ZG_EINVAL, std::string("relation/permission `") + perm + "` not found under definition `" + res_type + "`");
    if (!none_rel(subj_rel)) {
      int s = sc.slot_id(st, subj_rel);
      if (s < 0) return fail(ZG_EINVAL, std::string("relation `") + subj_rel + "` not found under definition `" + subj_type + "`");
      sr = static_cast<uint16_t>(s);
    }
    res = e->store.find(rt, res_id);
  }
  Device::SubjectsAnswer ans;
  if (res == ZG_NO_OBJECT) {
    // never written: no relationship names the resource. The engine state is still checked as for any lookup.
    if (wildcard_option != ZG_WILDCARDS_INCLUDE && wildcard_option != ZG_WILDCARDS_EXCLUDE)
      return fail(ZG_EINVAL, "unknown wildcard option");
    if (int rc = refuse(e, Call::kSubjects)) return rc;
  } else if (int rc = lookup_subjects_ids(e, static_cast<uint16_t>(p), res, static_cast<uint16_t>(st), sr, wildcard_option,
                                          &ans)) {
    return rc;
  }
  if (e->resolve_hook) e->resolve_hook(e->resolve_hook_arg);
  // lines: concrete ids, then "*" and one "!<id>" per exclusion ('!' is outside SpiceDB's object-id charset)
  std::vector<std::string> lines;
  {
    LOCK_NAMES_SHARED(e);
    auto name = [&](uint32_t id) {
      std::string_view n;
      return e->store.name(st, id, &n) ? std::string(n) : std::to_string(id);
    };
    for (uint32_t id : ans.ids) lines.push_back(name(id));
    if (ans.wildcard) {
      lines.push_back("*");
      for (uint32_t id : ans.excluded) lines.push_back("!" + name(id));
    }
  }
  size_t total = 1;
  for (const auto& l : lines) total += l.size() + 1;
  if (need) *need = total;
  if (n_out) *n_out = lines.size();
  if (total > cap || !buf) return ZG_E2BIG;
  size_t w = 0;
  for (const auto& l : lines) {
    std::memcpy(buf + w, l.data(), l.size());
    w += l.size();
    buf[w++] = '\n';
  }
  buf[w] = 0;
  return ZG_OK;
}

extern "C" int zg_lookup_subjects_str(zg_engine* e, const char* res_type, const char* res_id, const char* perm,
                                      const char* subj_type, const char* subj_rel, uint32_t wildcard_option, char* buf,
                                      size_t cap, size_t* need, uint64_t* n_out) {
  return with_stable_names(e, [&] {
    return lookup_subjects_str_once(e, res_type, res_id, perm, subj_type, subj_rel, wildcard_option, buf, cap, need,
                                    n_out);
  });
}

extern "C" int zg_lookup_subjects_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  out[0] = e->dev.subject_lookups_walk;
  out[1] = e->dev.subject_lookups_exhaustive;
  out[2] = e->dev.subject_items_verified;
  return ZG_OK;
}

// ExpandPermissionTree (Device::expand). Arguments are checked before anything else, against the ids handed out so far
// (a host-only engine still reports ZG_EINVAL for them); then, as for LookupSubjects, the device lock (FIFO), pending
// writes published, and the first device answers at the engine's clock.
static int expand_ids(zg_engine* e, const zg_expand_request* reqs, uint64_t n, std::vector<int32_t>* status,
                      std::vector<zg_expand_node>* nodes, std::vector<zg_expand_subject>* subjects) {
  const Schema& sc = e->schema;
  std::vector<Device::ExpandReq> xr(n);
  {
    LOCK_NAMES_SHARED(e);
    for (uint64_t i = 0; i < n; ++i) {
      const zg_expand_request& r = reqs[i];
      if (r.perm >= sc.slots.size()) return fail(ZG_EINVAL, "request " + std::to_string(i) + ": unknown relation or permission");
      const SlotInfo& si = sc.slots[r.perm];
      const std::string what = sc.types[si.type].name + "#" + si.name;
      if (!sc.x_ok[r.perm])
        return fail(ZG_EINVAL, "request " + std::to_string(i) + ": the tree of " + what + " has more than " +
                                   std::to_string(kMaxExpandTemplate) + " nodes per object");
      if (r.res != ZG_NO_OBJECT && r.res >= std::max(e->store.capacity(si.type), e->store.extent(si.type)))
        return fail(ZG_EINVAL, "request " + std::to_string(i) + ": object id " + std::to_string(r.res) +
                                   " is past the capacity of " + sc.types[si.type].name);
      xr[i] = Device::ExpandReq{r.res, sc.x_root[r.perm], sc.x_nodes[sc.x_root[r.perm]].ncount};
    }
  }
  if (int rc = refuse(e, Call::kExpand)) return rc;
  uint64_t cap = 1ull << 26;
  if (const char* v = std::getenv("ZGPU_EXPAND_CAP")) cap = std::strtoull(v, nullptr, 10);
  LOCK_DEVICE(e);
  if (e->dirty.load() || !e->dev.snap) {
    LOCK_NAMES_UNIQUE(e);
    int rc = publish_locked(e);
    if (rc) return rc;
  }
  e->dev.now = now_of(e);
  std::string err;
  const int rc = e->dev.expand(xr, cap, nodes, subjects, status, &err);
  return rc ? fail(rc, err) : ZG_OK;
}

extern "C" int zg_expand_permission_trees(zg_engine* e, const zg_expand_request* reqs, uint64_t n, int32_t* status,
                                          zg_expand_node* nodes, uint64_t node_cap, uint64_t* n_nodes,
                                          zg_expand_subject* subjects, uint64_t subj_cap, uint64_t* n_subjects) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!n_nodes || !n_subjects || (n && (!reqs || !status))) return fail(ZG_EINVAL, "NULL argument");
  std::vector<int32_t> st;
  std::vector<zg_expand_node> nv;
  std::vector<zg_expand_subject> sv;
  if (int rc = expand_ids(e, reqs, n, &st, &nv, &sv)) return rc;
  *n_nodes = nv.size();
  *n_subjects = sv.size();
  if (nv.size() > node_cap || sv.size() > subj_cap || (!nodes && !nv.empty()) || (!subjects && !sv.empty()))
    return fail(ZG_E2BIG, "output buffers too small");
  if (n) std::memcpy(status, st.data(), n * sizeof(int32_t));
  if (!nv.empty()) std::memcpy(nodes, nv.data(), nv.size() * sizeof(zg_expand_node));
  if (!sv.empty()) std::memcpy(subjects, sv.data(), sv.size() * sizeof(zg_expand_subject));
  return ZG_OK;
}

static int expand_str_once(zg_engine* e, const char* res_type, const char* res_id, const char* perm, char* buf, size_t cap,
                           size_t* need, uint64_t* n_lines) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!res_type || !res_id || !perm) return fail(ZG_EINVAL, "NULL argument");
  zg_expand_request r{};
  {
    LOCK_NAMES_SHARED(e);
    const Schema& sc = e->schema;
    const int rt = sc.type_id(res_type);
    if (rt < 0) return fail(ZG_EINVAL, std::string("object definition `") + res_type + "` not found");
    const int p = sc.slot_id(rt, perm);
    if (p < 0) return fail(ZG_EINVAL, std::string("relation/permission `") + perm + "` not found under definition `" + res_type + "`");
    r.perm = static_cast<uint16_t>(p);
    r.res = e->store.find(rt, res_id);
  }
  std::vector<int32_t> st;
  std::vector<zg_expand_node> nv;
  std::vector<zg_expand_subject> sv;
  if (int rc = expand_ids(e, &r, 1, &st, &nv, &sv)) return rc;
  if (st[0] == ZG_EDEPTH)
    return fail(ZG_EDEPTH, std::string("ExpandPermissionTree: the tree of ") + res_type + ":" + res_id + "#" + perm +
                               " passes the maximum depth (" + std::to_string(ZG_MAX_DEPTH) + " arrow hops)");
  if (e->resolve_hook) e->resolve_hook(e->resolve_hook_arg);
  // children in rank order; a parent precedes its children, so one pass fills every list
  std::vector<std::vector<uint32_t>> kids(nv.size());
  for (size_t i = 0; i < nv.size(); ++i)
    if (nv[i].parent != UINT32_MAX) {
      auto& k = kids[nv[i].parent];
      if (k.size() <= nv[i].rank) k.resize(nv[i].rank + 1, UINT32_MAX);
      k[nv[i].rank] = static_cast<uint32_t>(i);
    }
  std::string out;
  {
    LOCK_NAMES_SHARED(e);
    const Schema& sc = e->schema;
    auto name = [&](int t, uint32_t id) {
      if (id == ZG_NO_OBJECT) return std::string(res_id);  // the never-written resource and its same-object nodes
      std::string_view n;
      return e->store.name(t, id, &n) ? std::string(n) : std::to_string(id);
    };
    static const char kOp[] = "?UIXL";
    std::vector<std::pair<uint32_t, uint32_t>> stack;  // node, depth
    if (!nv.empty()) stack.push_back({0, 0});
    while (!stack.empty()) {
      const auto [i, d] = stack.back();
      stack.pop_back();
      const zg_expand_node& o = nv[i];
      const SlotInfo& si = sc.slots[o.slot];
      out += std::to_string(d) + " " + kOp[o.op <= 4 ? o.op : 0] + " " + sc.types[si.type].name + ":" + name(si.type, o.object) +
             "#" + si.name;
      for (uint64_t j = o.subjects; j < o.subjects + o.n_subjects; ++j) {
        const zg_expand_subject& x = sv[j];
        out += " " + sc.types[x.type].name + ":" + (x.srel == kWildcard ? std::string("*") : name(x.type, x.id));
        if (x.srel != kWildcard && x.srel != kNone) out += "#" + sc.slots[x.srel].name;
      }
      out += "\n";
      for (auto it = kids[i].rbegin(); it != kids[i].rend(); ++it) stack.push_back({*it, d + 1});
    }
  }
  if (need) *need = out.size() + 1;
  if (n_lines) *n_lines = nv.size();
  if (out.size() + 1 > cap || !buf) return fail(ZG_E2BIG, "output buffer too small");
  std::memcpy(buf, out.c_str(), out.size() + 1);
  return ZG_OK;
}

extern "C" int zg_expand_permission_tree_str(zg_engine* e, const char* res_type, const char* res_id, const char* perm,
                                             char* buf, size_t cap, size_t* need, uint64_t* n_lines) {
  return with_stable_names(e, [&] { return expand_str_once(e, res_type, res_id, perm, buf, cap, need, n_lines); });
}

extern "C" int zg_expand_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  out[0] = e->dev.x_trees;
  out[1] = e->dev.x_levels;
  out[2] = e->dev.x_nodes_out;
  out[3] = e->dev.x_subjects_out;
  return ZG_OK;
}

extern "C" int zg_expand_last_times(zg_engine* e, double* ms, uint64_t cap, uint64_t* n) {
  if (!e || !n) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto& t = e->dev.x_last_ms;
  *n = t.size();
  if (t.size() > cap || (!ms && !t.empty())) return fail(ZG_E2BIG, "output buffer too small");
  if (!t.empty()) std::memcpy(ms, t.data(), t.size() * sizeof(double));
  return ZG_OK;
}

extern "C" int zg_closure_index_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  uint64_t c[7] = {0, 0, 0, 0, e->dev.closure_builds, static_cast<uint64_t>(e->dev.closure_ms * 1000.0),
                   e->dev.closure_failures};
  if (const auto s = e->dev.snap)
    for (const auto& x : s->closure) {
      ++c[x.built ? 0 : 1];
      c[2] += x.entries;
      c[3] += x.row_ptr.cap + x.col.cap;
    }
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_closure_index_copy(zg_engine* e, uint32_t pair, uint32_t* row_ptr, uint64_t row_cap, uint32_t* col,
                                     uint64_t col_cap, uint64_t* n_rows, uint64_t* n_entries) {
  if (!e || !n_rows || !n_entries) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto s = e->dev.snap;
  if (!s) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
  if (pair >= s->closure.size() || !s->closure[pair].built) return fail(ZG_EINVAL, "no closure index for this pair");
  const auto& x = s->closure[pair];
  *n_rows = x.nsubj;
  *n_entries = x.entries;
  if (row_cap < uint64_t(x.nsubj) + 1 || col_cap < x.entries || !row_ptr || (!col && x.entries))
    return fail(ZG_E2BIG, "buffers too small for the closure index");
  cudaError_t ce = cudaSetDevice(e->dev.device);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->dev.stream);
  if (ce == cudaSuccess) ce = cudaMemcpy(row_ptr, x.row_ptr.p, (uint64_t(x.nsubj) + 1) * 4, cudaMemcpyDeviceToHost);
  if (ce == cudaSuccess && x.entries) ce = cudaMemcpy(col, x.col.p, x.entries * x.width, cudaMemcpyDeviceToHost);
  if (ce == cudaSuccess && x.width == 2) {
    // widened in place from the back: entry i (bytes 2i ..) is read before word i (bytes 4i ..) is written
    const uint16_t* narrow = reinterpret_cast<const uint16_t*>(col);
    for (uint64_t i = x.entries; i-- > 0;) col[i] = narrow[i];
  }
  return ce == cudaSuccess ? ZG_OK : fail(ZG_ECUDA, std::string("zg_closure_index_copy: ") + cudaGetErrorString(ce));
}

extern "C" int zg_closure_index_info(zg_engine* e, uint32_t pair, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto s = e->dev.snap;
  if (!s) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
  if (pair >= s->closure.size()) return fail(ZG_EINVAL, "no two-level pair with this number");
  const auto& x = s->closure[pair];
  const uint64_t c[4] = {x.built ? 1u : 0u, x.built ? x.width : 0u, x.entries, x.built ? x.row_ptr.cap + x.col.cap : 0u};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_closure_signature_info(zg_engine* e, uint32_t pair, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto s = e->dev.snap;
  if (!s) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
  if (pair >= s->closure.size()) return fail(ZG_EINVAL, "no two-level pair with this number");
  const auto& x = s->closure[pair];
  const bool b = x.built && x.sig_words;
  const uint64_t c[5] = {b ? 1u : 0u, b ? x.sig_words : 0u, b ? 3u : 0u, b ? uint64_t(x.nsubj) * x.sig_words * 8 : 0u,
                         b ? static_cast<uint64_t>(x.sig_ms * 1000.0) : 0u};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_closure_signature_copy(zg_engine* e, uint32_t pair, uint64_t* words, uint64_t cap, uint64_t* n_words) {
  if (!e || !n_words) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto s = e->dev.snap;
  if (!s) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
  if (pair >= s->closure.size() || !s->closure[pair].built || !s->closure[pair].sig_words)
    return fail(ZG_EINVAL, "no closure signatures for this pair");
  const auto& x = s->closure[pair];
  *n_words = uint64_t(x.nsubj) * x.sig_words;
  if (cap < *n_words || (!words && *n_words)) return fail(ZG_E2BIG, "buffer too small for the closure signatures");
  cudaError_t ce = cudaSetDevice(e->dev.device);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->dev.stream);
  if (ce == cudaSuccess && *n_words) ce = cudaMemcpy(words, x.sig.p, *n_words * 8, cudaMemcpyDeviceToHost);
  return ce == cudaSuccess ? ZG_OK : fail(ZG_ECUDA, std::string("zg_closure_signature_copy: ") + cudaGetErrorString(ce));
}

extern "C" int zg_closure_table_info(zg_engine* e, uint32_t pair, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto s = e->dev.snap;
  if (!s) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
  if (pair >= s->closure.size()) return fail(ZG_EINVAL, "no two-level pair with this number");
  const auto& x = s->closure[pair];
  const bool b = x.built && x.set_built;
  const uint64_t c[5] = {b ? 1u : 0u, b ? x.set_buckets : 0u, b ? zg::kTableSlots : 0u,
                         b ? (uint64_t(x.nsubj) + x.set_buckets) * 8 : 0u, b ? static_cast<uint64_t>(x.set_ms * 1000.0) : 0u};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_closure_table_copy(zg_engine* e, uint32_t pair, uint64_t* hdr, uint64_t hdr_cap, uint64_t* buckets,
                                     uint64_t bucket_cap, uint64_t* n_rows, uint64_t* n_buckets) {
  if (!e || !n_rows || !n_buckets) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto s = e->dev.snap;
  if (!s) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
  if (pair >= s->closure.size() || !s->closure[pair].built || !s->closure[pair].set_built)
    return fail(ZG_EINVAL, "no closure set table for this pair");
  const auto& x = s->closure[pair];
  *n_rows = x.nsubj;
  *n_buckets = x.set_buckets;
  if (hdr_cap < *n_rows || bucket_cap < *n_buckets || (!hdr && *n_rows) || (!buckets && *n_buckets))
    return fail(ZG_E2BIG, "buffer too small for the closure set table");
  cudaError_t ce = cudaSetDevice(e->dev.device);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->dev.stream);
  if (ce == cudaSuccess && *n_rows) ce = cudaMemcpy(hdr, x.set_hdr.p, *n_rows * 8, cudaMemcpyDeviceToHost);
  if (ce == cudaSuccess && *n_buckets) ce = cudaMemcpy(buckets, x.set_tab.p, *n_buckets * 8, cudaMemcpyDeviceToHost);
  return ce == cudaSuccess ? ZG_OK : fail(ZG_ECUDA, std::string("zg_closure_table_copy: ") + cudaGetErrorString(ce));
}

extern "C" int zg_flat_record_info(zg_engine* e, uint32_t k, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto s = e->dev.snap;
  if (!s) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
  if (k >= s->records.size()) return fail(ZG_EINVAL, "no range records with this number");
  const auto& r = s->records[k];
  const bool b = r.built;
  const uint64_t c[6] = {b ? 1u : 0u, r.gc, r.nres, b ? uint64_t(r.nres) * zg::kRecSlots * 2 : 0u, b ? r.long_rows : 0u,
                         b ? static_cast<uint64_t>(r.ms * 1000.0) : 0u};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_flat_record_copy(zg_engine* e, uint32_t k, uint16_t* slots, uint64_t cap, uint64_t* n_slots) {
  if (!e || !n_slots) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const auto s = e->dev.snap;
  if (!s) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
  if (k >= s->records.size() || !s->records[k].built) return fail(ZG_EINVAL, "no range records with this number");
  const auto& r = s->records[k];
  *n_slots = uint64_t(r.nres) * zg::kRecSlots;
  if (cap < *n_slots || (!slots && *n_slots)) return fail(ZG_E2BIG, "buffer too small for the range records");
  cudaError_t ce = cudaSetDevice(e->dev.device);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->dev.stream);
  if (ce == cudaSuccess && *n_slots) ce = cudaMemcpy(slots, r.rec.p, *n_slots * 2, cudaMemcpyDeviceToHost);
  return ce == cudaSuccess ? ZG_OK : fail(ZG_ECUDA, std::string("zg_flat_record_copy: ") + cudaGetErrorString(ce));
}

extern "C" int zg_handle_lookup_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const uint64_t c[7] = {e->hl_rounds, e->hl_levels, e->hl_round_trips, e->hl_frontier, e->hl_candidates, e->hl_halvings,
                         e->hl_fallbacks};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_handle_subjects_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  LOCK_DEVICE(e);
  const uint64_t c[7] = {e->hs_lookups, e->hs_levels, e->hs_waits, e->hs_entries, e->hs_candidates, e->hs_nowild,
                         e->hs_fallbacks};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

extern "C" int zg_filter_counters(zg_engine* e, uint64_t* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  const uint64_t c[6] = {e->flt_device.load(), e->flt_host.load(), e->flt_returned.load(),
                         e->flt_shape[Device::kByResource].load(), e->flt_shape[Device::kBySubject].load(),
                         e->flt_shape[Device::kByScan].load()};
  std::memcpy(out, c, sizeof c);
  return ZG_OK;
}

// ---- pre-filter: LookupResources ids -> kept list items --------------------------------------

extern "C" int zg_list_keep_allowed(zg_engine* e, const char* body, size_t len, const zg_list_item* items, uint64_t n,
                                    uint32_t mode, const char* res_type, const char* req_namespace, const uint32_t* allowed,
                                    uint64_t n_allowed, const char* self_name, uint8_t* keep) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!res_type || ((!body || !items || !keep) && n) || (!allowed && n_allowed)) return fail(ZG_EINVAL, "NULL argument");
  if (mode > ZG_LIST_PROTOBUF) return fail(ZG_EINVAL, "unknown mode");
  LOCK_NAMES_SHARED(e);
  const int rt = e->schema.type_id(res_type);
  if (rt < 0) return fail(ZG_EINVAL, std::string("object definition `") + res_type + "` not found");
  const std::string req_ns = req_namespace ? req_namespace : "", self = self_name ? self_name : "";
  auto has = [&](const std::string& id) {
    if (!self.empty() && id == self) return true;
    const uint32_t oid = e->store.find(rt, id.data(), id.size());
    return oid != ZG_NO_OBJECT && std::binary_search(allowed, allowed + n_allowed, oid);
  };
  std::string name, ns, id;
  for (uint64_t i = 0; i < n; ++i) {
    const zg_list_item& it = items[i];
    keep[i] = 0;
    if (!(it.flags & ZG_ITEM_IS_OBJECT)) return fail(ZG_EINVAL, "failed to decode response body: element is not an object");
    if (mode == ZG_LIST_TABLE_ROWS && !(it.flags & ZG_ITEM_HAS_OBJECT))
      return fail(ZG_EINVAL, "error decoding partial object metadata from table row");
    if (it.name_off > len || it.name_len > len - it.name_off || it.ns_off > len || it.ns_len > len - it.ns_off)
      return fail(ZG_EINVAL, "item range outside the body");
    name.clear();
    ns.clear();
    if ((it.flags & ZG_ITEM_HAS_METADATA) && (it.flags & ZG_ITEM_RAW_NAMES)) {
      name.assign(body + it.name_off, it.name_len);  // protobuf strings: plain bytes
      ns.assign(body + it.ns_off, it.ns_len);
    } else if (it.flags & ZG_ITEM_HAS_METADATA) {
      json_unescape_append(body + it.name_off, it.name_len, &name);
      json_unescape_append(body + it.ns_off, it.ns_len, &ns);
    }
    // an allowed id maps to (text before the last '/', text after it): a name holding a '/' maps from none
    if (name.empty() || name.find('/') != std::string::npos) continue;
    id = ns;
    id += '/';
    id += name;
    bool k = has(id);
    if (!k && ns == req_ns) k = has(name);  // cluster-scoped ids take the request's namespace (lookups.go:117-127)
    keep[i] = k ? 1 : 0;
  }
  return ZG_OK;
}

static int list_prefilter_once(zg_engine* e, const char* body, size_t len, uint32_t mode, const zg_list_template* tpl,
                               char* out, size_t cap, size_t* out_len) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!body || !out_len || !tpl) return fail(ZG_EINVAL, "NULL argument");
  if (!tpl->res_type || !tpl->permission || !tpl->subj_type || !tpl->subj_id) return fail(ZG_EINVAL, "NULL template field");
  if (mode > ZG_LIST_PROTOBUF) return fail(ZG_EINVAL, "unknown mode");
  if (int rc = refuse(e, Call::kLookup)) return rc;
  // 1. the allowed ids (one LookupResources on the GPU; concurrent list requests share launches)
  std::vector<uint32_t> ids;
  std::string self;
  int rt = -1;
  {
    int p, st;
    uint16_t sr;
    uint32_t su;
    int rc = resolve_lookup_strs(e, tpl->res_type, tpl->permission, tpl->subj_type, tpl->subj_id, tpl->subj_rel, &rt, &p, &st,
                                 &sr, &su);
    if (rc) return rc;
    bool self_member = false;
    rc = lookup_queued(e, static_cast<uint16_t>(rt), static_cast<uint16_t>(p), static_cast<uint16_t>(st),
                       su == ZG_NO_OBJECT ? ZG_NO_OBJECT - 1 : su, sr, &ids, &self_member);
    if (rc) return rc;
    if (su == ZG_NO_OBJECT && self_member) self = tpl->subj_id;  // never-written userset subject naming itself
    // lookups.go:106-109: an id that yields no name fails the whole pre-filter
    LOCK_NAMES_SHARED(e);
    for (uint32_t id : ids) {
      std::string_view nm;
      if (e->store.name(rt, id, &nm) && nm.back() == '/') return fail(ZG_EINVAL, "unable to determine name for resource");
    }
  }
  // 2. scan
  size_t icap = len / 128 + 16;
  std::unique_ptr<zg_list_item[]> items(new (std::nothrow) zg_list_item[icap]);
  if (!items) return fail(ZG_ENOMEM, "out of host memory");
  uint64_t ib = 0, ie = 0;
  int64_t n = zg_list_scan(body, len, mode, items.get(), icap, &ib, &ie);
  if (n == ZG_E2BIG) {
    n = zg_list_scan(body, len, mode, nullptr, 0, &ib, &ie);
    if (n > 0) {
      icap = static_cast<size_t>(n);
      items.reset(new (std::nothrow) zg_list_item[icap]);
      if (!items) return fail(ZG_ENOMEM, "out of host memory");
      n = zg_list_scan(body, len, mode, items.get(), icap, &ib, &ie);
    }
  }
  if (n < 0) return fail(ZG_EINVAL, "failed to decode response body");
  if (ie == 0) {  // no such array: the body passes through
    *out_len = len;
    if (len > cap || !out) return ZG_E2BIG;
    std::memcpy(out, body, len);
    return ZG_OK;
  }
  // 3. keep + splice
  const uint64_t N = static_cast<uint64_t>(n);
  std::vector<uint8_t> keep(N);
  int rc = zg_list_keep_allowed(e, body, len, items.get(), N, mode, tpl->res_type, tpl->req_namespace, ids.data(), ids.size(),
                                self.empty() ? nullptr : self.c_str(), keep.data());
  if (rc) return rc;
  rc = zg_list_filter(body, len, items.get(), N, keep.data(), ib, ie, 0, out, cap, out_len);
  return rc == ZG_EINVAL ? fail(rc, "zg_list_filter: inconsistent item ranges") : rc;
}

extern "C" int zg_list_prefilter(zg_engine* e, const char* body, size_t len, uint32_t mode, const zg_list_template* tpl,
                                 char* out, size_t cap, size_t* out_len) {
  return with_stable_names(e, [&] { return list_prefilter_once(e, body, len, mode, tpl, out, cap, out_len); });
}

extern "C" int zg_stats_get(zg_engine* e, zg_stats* out) {
  if (!e || !out) return fail(ZG_EINVAL, "NULL argument");
  std::lock_guard<FairMutex> g(e->mu);
  if (!e->host_only) e->dev.finish_timing();
  std::memset(out, 0, sizeof *out);
  out->checks = e->dev.checks;
  out->launches = e->dev.launches;
  out->passes = e->dev.passes;
  out->revision = e->revision;
  out->last_alg_bytes = e->dev.last_alg_bytes;
  out->last_kernel_ms = e->dev.last_ms;
  out->coalesced_launches = e->dev.coalesced_launches;
  out->coalesced_requests = e->dev.coalesced_requests;
  out->split_batches = e->dev.split_batches;
  out->delta_publishes = e->dev.delta_publishes;
  out->full_publishes = e->dev.full_publishes;
  out->last_publish_ms = e->dev.last_build_ms;
  out->streamed_calls = e->dev.streamed_calls;
  out->lookup_batches = e->dev.lookup_batches;
  out->lookups_batched = e->dev.lookups_batched;
  if (!e->host_only) e->dev.read_events(&out->stack_spills, &out->memo_batches);
  out->devices = is_handle(e) ? e->shard_devices : 1 + e->replicas.size();
  out->shards = e->n_shards;
  out->last_levels = e->last_group.levels;
  out->last_subqueries = e->last_group.subqueries;
  out->last_round_trips = e->last_group.round_trips;
  for (auto& r : e->replicas) {
    const Device& d = r->dev;
    out->checks += d.checks;
    out->launches += d.launches;
    out->passes += d.passes;
    out->split_batches += d.split_batches;
    out->delta_publishes += d.delta_publishes;
    out->full_publishes += d.full_publishes;
    out->streamed_calls += d.streamed_calls;
    out->lookup_batches += d.lookup_batches;
    out->lookups_batched += d.lookups_batched;
  }
  if (e->dev.snap) {
    out->tuples = e->dev.snap->n_tuples;
    out->snapshot_bytes = e->dev.snap->bytes;
    out->flat_slots = e->dev.snap->flat_slots;
  }
  if (!e->host_only) out->flat_residual = e->dev.flat_residual();
  for (uint32_t k = 1; k < e->n_shards && !e->host_only; ++k)  // a sharded handle: every shard's part
    if (const auto s = shard(e, k).snap) {
      out->tuples += s->n_tuples;
      out->snapshot_bytes += s->bytes;
    }
  return ZG_OK;
}

// ---- sharded store, device-resident protocol (no host staging between passes) ----
#define SHARD_PROLOGUE()                                                                                              \
  NEED_SCHEMA(e, ZG_ENOSCHEMA);                                                                                       \
  std::lock_guard<FairMutex> g(e->mu);                                                                               \
  if (int rc_ = refuse(e, Call::kShardCall)) return rc_;                                                             \
  if (!e->dev.snap) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");

extern "C" int zg_shard_route_dev(zg_engine* e, const zg_check* d_items, uint64_t n, int level, uint32_t n_dest,
                                  zg_check* d_routed, uint32_t* d_src, uint64_t* counts) {
  if (!counts || ((!d_routed || !d_src) && n)) return fail(ZG_EINVAL, "NULL argument");
  SHARD_PROLOGUE();
  std::string err;
  int rc = e->dev.route_by_owner(d_items, n, level, n_dest, d_routed, d_src, counts, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_pass_dev(zg_engine* e, const zg_check* d_queries, uint64_t n, int level, uint64_t* n_sub) {
  if ((!d_queries && n) || !n_sub || level < 0 || level > ZG_MAX_DEPTH + 2) return fail(ZG_EINVAL, "bad argument");
  SHARD_PROLOGUE();
  e->dev.now = now_of(e);
  std::string err;
  int rc = e->dev.shard_pass_dev(d_queries, n, level, n_sub, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_fold_dev(zg_engine* e, int level, const uint8_t* d_child_vals, const uint32_t* d_src, uint64_t n_sub,
                                 uint8_t* d_out, int final_codes) {
  if (((!d_child_vals || !d_src) && n_sub) || level < 0) return fail(ZG_EINVAL, "bad argument");
  SHARD_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_fold_dev(level, d_child_vals, d_src, n_sub, d_out, final_codes != 0, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_unroute_dev(zg_engine* e, const uint32_t* d_src, const uint8_t* d_val, uint64_t n, uint8_t* d_out) {
  if ((!d_src || !d_val || !d_out) && n) return fail(ZG_EINVAL, "NULL argument");
  SHARD_PROLOGUE();
  std::string err;
  int rc = e->dev.unroute(d_src, d_val, n, d_out, &err);
  return rc ? fail(rc, err) : ZG_OK;
}

// LookupResources / LookupSubjects on the sharded store: the same prologue, and only on a sharded engine (the
// message names the unsharded call)
#define SHARD_ONLY_PROLOGUE(unsharded_msg)                                                                            \
  NEED_SCHEMA(e, ZG_ENOSCHEMA);                                                                                       \
  std::lock_guard<FairMutex> g(e->mu);                                                                               \
  if (int rc_ = refuse(e, Call::kShardCall)) return rc_;                                                             \
  if (e->dev.shard_count < 2) return fail(ZG_EINVAL, unsharded_msg);                                                 \
  if (!e->dev.snap) return fail(ZG_ENOSNAPSHOT, "no snapshot published (call zg_publish)");
#define SHARD_LOOKUP_PROLOGUE() SHARD_ONLY_PROLOGUE("not a sharded engine: use zg_lookup_resources")
#define SHARD_SUBJECTS_PROLOGUE() SHARD_ONLY_PROLOGUE("not a sharded engine: use zg_lookup_subjects")

extern "C" int zg_shard_lookup_begin_dev(zg_engine* e, const uint16_t* res_types, const zg_check* protos, const uint8_t* home,
                                         uint32_t k, uint64_t walk_cap, uint64_t* d_seeds) {
  if (!res_types || !protos || !home || !d_seeds) return fail(ZG_EINVAL, "NULL argument");
  SHARD_LOOKUP_PROLOGUE();
  std::vector<Device::LookupReq> reqs(k);
  for (uint32_t i = 0; i < k; ++i) reqs[i] = Device::LookupReq{res_types[i], protos[i]};
  std::string err;
  int rc = e->dev.shard_lookup_begin(reqs, home, walk_cap, reinterpret_cast<unsigned long long*>(d_seeds), &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_lookup_expand_dev(zg_engine* e, const uint64_t* d_front, uint64_t n_in, int level, uint64_t* d_next,
                                          uint64_t* n_next, int* overflow) {
  if ((!d_front && n_in) || !d_next || !n_next || !overflow) return fail(ZG_EINVAL, "NULL argument");
  SHARD_LOOKUP_PROLOGUE();
  std::string err;
  bool ovf = false;
  int rc = e->dev.shard_lookup_expand(reinterpret_cast<const unsigned long long*>(d_front), n_in, level,
                                      reinterpret_cast<unsigned long long*>(d_next), n_next, &ovf, &err);
  *overflow = ovf ? 1 : 0;
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_lookup_candidates_dev(zg_engine* e, int exhaustive, zg_check* d_items, uint64_t cap, uint64_t* n) {
  if (!n) return fail(ZG_EINVAL, "NULL argument");
  SHARD_LOOKUP_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_lookup_candidates(exhaustive != 0, d_items, cap, n, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_lookup_route_dev(zg_engine* e, const uint8_t* d_codes, uint64_t n, uint32_t n_dest, uint64_t* d_routed,
                                         uint64_t* counts) {
  if (!counts || ((!d_codes || !d_routed) && n)) return fail(ZG_EINVAL, "NULL argument");
  SHARD_LOOKUP_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_lookup_route(d_codes, n, n_dest, reinterpret_cast<unsigned long long*>(d_routed), counts, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_lookup_finish_dev(zg_engine* e, const uint64_t* d_keys, uint64_t n, uint32_t* d_ids, uint64_t* per_lookup,
                                          uint64_t* err_mask) {
  if (!per_lookup || !err_mask || ((!d_keys || !d_ids) && n)) return fail(ZG_EINVAL, "NULL argument");
  SHARD_LOOKUP_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_lookup_finish(reinterpret_cast<const unsigned long long*>(d_keys), n, d_ids, per_lookup, err_mask, &err);
  return rc ? fail(rc, err) : ZG_OK;
}

// LookupSubjects on the sharded store
extern "C" int zg_shard_pass_nowild_dev(zg_engine* e, const zg_check* d_queries, uint64_t n, int level, uint64_t* n_sub) {
  if ((!d_queries && n) || !n_sub || level < 0 || level > ZG_MAX_DEPTH + 2) return fail(ZG_EINVAL, "bad argument");
  SHARD_SUBJECTS_PROLOGUE();
  e->dev.now = now_of(e);
  std::string err;
  int rc = e->dev.shard_pass_nowild_dev(d_queries, n, level, n_sub, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_subjects_begin_dev(zg_engine* e, const uint16_t* res_types, const zg_check* reqs, const uint32_t* options,
                                           const uint8_t* home, uint32_t k, uint64_t walk_cap, uint64_t* d_front, uint64_t* n_front) {
  if (!res_types || !reqs || !options || !home || !d_front || !n_front) return fail(ZG_EINVAL, "NULL argument");
  SHARD_SUBJECTS_PROLOGUE();
  const Schema& sc = e->schema;
  std::vector<Device::SubjectsReq> rs(k);
  uint64_t include = 0;
  for (uint32_t i = 0; i < k; ++i) {
    const zg_check& q = reqs[i];
    // as zg_lookup_subjects (the permission's slot also bounds the walk's mask read)
    if (q.perm >= sc.slots.size() || sc.slots[q.perm].type != res_types[i]) return fail(ZG_EINVAL, "unknown permission of the resource type");
    if (q.stype >= sc.types.size() || (q.srel != kNone && (q.srel >= sc.slots.size() || sc.slots[q.srel].type != q.stype)))
      return fail(ZG_EINVAL, "unknown subject type or relation");
    if (options[i] != ZG_WILDCARDS_INCLUDE && options[i] != ZG_WILDCARDS_EXCLUDE) return fail(ZG_EINVAL, "unknown wildcard option");
    rs[i] = Device::SubjectsReq{q.res, res_types[i], q.perm, q.stype, q.srel};
    if (options[i] == ZG_WILDCARDS_INCLUDE && i < 64) include |= 1ull << i;
  }
  std::string err;
  int rc = e->dev.shard_subjects_begin(rs, home, include, walk_cap, reinterpret_cast<unsigned long long*>(d_front), n_front, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_subjects_expand_dev(zg_engine* e, const uint64_t* d_front, uint64_t n_in, uint32_t n_dest, uint64_t* d_routed,
                                            uint64_t* counts, int* overflow) {
  if ((!d_front && n_in) || !d_routed || !counts || !overflow) return fail(ZG_EINVAL, "NULL argument");
  SHARD_SUBJECTS_PROLOGUE();
  std::string err;
  bool ovf = false;
  int rc = e->dev.shard_subjects_expand(reinterpret_cast<const unsigned long long*>(d_front), n_in, n_dest,
                                        reinterpret_cast<unsigned long long*>(d_routed), counts, &ovf, &err);
  *overflow = ovf ? 1 : 0;
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_subjects_admit_dev(zg_engine* e, const uint64_t* d_in, uint64_t n_in, uint64_t* d_next, uint64_t* n_next) {
  if ((!d_in && n_in) || !d_next || !n_next) return fail(ZG_EINVAL, "NULL argument");
  SHARD_SUBJECTS_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_subjects_admit(reinterpret_cast<const unsigned long long*>(d_in), n_in, reinterpret_cast<unsigned long long*>(d_next),
                                       n_next, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_subjects_candidates_dev(zg_engine* e, int exhaustive, zg_check* d_items, uint64_t cap, uint64_t* n) {
  if (!n) return fail(ZG_EINVAL, "NULL argument");
  SHARD_SUBJECTS_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_subjects_candidates(exhaustive != 0, d_items, cap, n, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_subjects_verdicts_dev(zg_engine* e, const uint8_t* d_codes, uint64_t n, uint64_t* granted, uint64_t* failed) {
  if ((!d_codes && n) || !granted || !failed) return fail(ZG_EINVAL, "NULL argument");
  SHARD_SUBJECTS_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_subjects_verdicts(d_codes, n, granted, failed, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_subjects_nowild_dev(zg_engine* e, const uint8_t* d_codes, uint64_t n, uint64_t granted, uint64_t failed,
                                            zg_check* d_items, uint64_t cap, uint64_t* n_nw) {
  if (((!d_codes || !d_items) && n) || !n_nw) return fail(ZG_EINVAL, "NULL argument");
  SHARD_SUBJECTS_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_subjects_nowild(d_codes, n, granted, failed, d_items, cap, n_nw, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_subjects_route_dev(zg_engine* e, const uint8_t* d_codes, uint64_t n, uint32_t n_dest, uint64_t* d_routed,
                                           uint64_t* counts) {
  if (!counts || !d_routed || (!d_codes && n)) return fail(ZG_EINVAL, "NULL argument");
  SHARD_SUBJECTS_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_subjects_route(d_codes, n, n_dest, reinterpret_cast<unsigned long long*>(d_routed), counts, &err);
  return rc ? fail(rc, err) : ZG_OK;
}
extern "C" int zg_shard_subjects_finish_dev(zg_engine* e, const uint64_t* d_keys, uint64_t n, uint32_t* d_ids, uint64_t* listed,
                                            uint64_t* excluded) {
  if (!listed || !excluded || ((!d_keys || !d_ids) && n)) return fail(ZG_EINVAL, "NULL argument");
  SHARD_SUBJECTS_PROLOGUE();
  std::string err;
  int rc = e->dev.shard_subjects_finish(reinterpret_cast<const unsigned long long*>(d_keys), n, d_ids, listed, excluded, &err);
  return rc ? fail(rc, err) : ZG_OK;
}

static int debug_row_of(const zg_engine* e, const HostSnapshot& h, uint16_t rel_slot, uint32_t res, uint32_t cls, uint32_t* out,
                        uint64_t cap, uint64_t* n_out) {
  const Schema& sc = e->schema;
  if (rel_slot >= sc.slots.size() || sc.slots[rel_slot].is_perm) return fail(ZG_EINVAL, "not a relation");
  const DRel& r = h.rels[sc.slots[rel_slot].rel_index];
  *n_out = 0;
  if (cls & 0x80000000u) {  // reverse row: `res` is the SUBJECT id, result = resources listing it
    cls &= 0x7FFFFFFFu;
    if (cls >= r.ncls) return fail(ZG_EINVAL, "class out of range");
    const DCls& c = h.cls[r.cls_begin + cls];
    const uint32_t row = c.sslot == kWildcard ? 0u : res;
    if (row >= c.nsubj) return ZG_OK;
    const uint64_t ri = c.rrow_base + uint64_t(row) * c.rstride;
    uint32_t b = h.rrow_ptr[ri], en = h.rrow_ptr[ri + 1];
    *n_out = en - b;
    if (en - b > cap) return ZG_E2BIG;
    for (uint32_t i = b; i < en; ++i) out[i - b] = h.rcol[i];
    return ZG_OK;
  }
  if (cls >= r.ncls) return fail(ZG_EINVAL, "class out of range");
  if (res >= r.nres) return ZG_OK;
  uint64_t idx = r.row_base + uint64_t(res) * r.stride + cls;
  uint32_t b = h.row_ptr[idx], en = h.row_ptr[idx + 1];
  *n_out = en - b;
  if (en - b > cap) return ZG_E2BIG;
  for (uint32_t i = b; i < en; ++i) out[i - b] = h.col[i];
  return ZG_OK;
}
extern "C" int zg_debug_row(zg_engine* e, uint16_t rel_slot, uint32_t res, uint32_t cls, uint32_t* out, uint64_t cap,
                            uint64_t* n_out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!n_out) return fail(ZG_EINVAL, "NULL n_out");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  e->keep_built = true;
  if (e->last_built.rels.empty() && !e->schema.rel_slots.empty()) {
    e->last_built = e->store.build();
    if (!e->last_built.err.empty()) return fail(ZG_EINVAL, e->last_built.err);
  }
  return debug_row_of(e, e->last_built, rel_slot, res, cls, out, cap, n_out);
}
extern "C" int zg_debug_shard_row(zg_engine* e, uint32_t shard, uint16_t rel_slot, uint32_t res, uint32_t cls, uint32_t* out,
                                  uint64_t cap, uint64_t* n_out) {
  NEED_SCHEMA(e, ZG_ENOSCHEMA);
  if (!n_out) return fail(ZG_EINVAL, "NULL n_out");
  if (!is_handle(e) || shard >= e->n_shards) return fail(ZG_EINVAL, "not a shard of a sharded handle (zg_config.n_shards)");
  LOCK_DEVICE(e);
  LOCK_NAMES_UNIQUE(e);
  if (e->shard_built.size() != e->n_shards) e->shard_built.assign(e->n_shards, HostSnapshot());
  HostSnapshot& h = e->shard_built[shard];
  if (h.rels.empty() && !e->schema.rel_slots.empty()) {
    h = e->store.build(shard, e->n_shards);
    if (!h.err.empty()) return fail(ZG_EINVAL, h.err);
  }
  return debug_row_of(e, h, rel_slot, res, cls, out, cap, n_out);
}

extern "C" const char* zg_build_info(void) { return zg::build_info(); }

extern "C" void* zg_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) {
    cudaGetLastError();
    g_err = "cudaMallocHost failed";
    return nullptr;
  }
  return p;
}
extern "C" void zg_host_free(void* p) {
  if (p) cudaFreeHost(p);
}
