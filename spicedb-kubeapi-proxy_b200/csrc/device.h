// device.h -- device-side state of one engine: the published CSR snapshot in HBM,
// scratch buffers, and the launch sequences of the hot path.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "../../include/zgpu.h"
#include "schema.h"
#include "store.h"

namespace zg {

struct FilterSel;   // filter.cuh
struct FilterPlan;

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  // grow-only; returns false on allocation failure
  bool ensure(size_t bytes);
  void release();
  template <class T>
  T* as() const { return static_cast<T*>(p); }
};

// Immutable once published; shared_ptr keeps it alive for in-flight readers.
struct Snapshot {
  DevBuf row_ptr, col, exp, prog, rrow_ptr, rcol, type_bit_base;
  // incremental publish (build.cu gpu_apply_delta): the edge arrays are re-emitted into their alternates and
  // swapped; per-class relationship counts tell when a class becomes (non-)empty and the program changes
  DevBuf col_alt, exp_alt, rcol_alt;
  std::vector<uint64_t> cls_count;
  std::vector<uint64_t> type_base;   // per type: first row_ptr index of its objects
  std::vector<uint32_t> type_ncls;   // per type: row stride
  bool delta_ok = false;             // built by the GPU builder: counts are known
  bool resources_stale = false;      // resources[] predate an incremental publish: rebuilt on first use
  std::vector<uint32_t> n_objects;  // per type
  std::vector<DRel> rels;           // the layout's row tables, for the host to plan from (Device::match_filter);
  std::vector<DCls> cls;            // the classes' CF_EMPTY flags are those of the last structural publish
  uint64_t total_bits = 0;          // visited bitmap size for the reverse BFS
  // Per slot: device array of FlatLookupClass when the slot is a flat union of direct
  // (non-expiring) relations; flat_n[slot] = -1 otherwise.
  std::vector<DevBuf> flat_cls;
  std::vector<int> flat_n;
  std::vector<DevBuf> resources;  // per type
  // LookupSubjects' forward walk: Schema::forward_tables / fwd_mask of this layout
  DevBuf ls_fwd, ls_type_off, ls_mask;
  uint32_t ls_mask_words = 1;
  // ExpandPermissionTree (expand.cuh): the schema's templates (Schema::x_*) and this layout's relation and class tables
  DevBuf x_nodes, x_tgts, x_counted, x_rels, x_cls;
  std::vector<uint64_t> n_resources;
  uint32_t prog_bytes = 0;
  uint32_t max_leaves = 1;
  bool has_nonpure = false;
  bool has_l2 = false;  // some step of the program meets two levels (kStepTargetL2)
  uint32_t flat_slots = 0;  // slots marked SF_FLAT at publish (mark_flat_slots): checks flat_check_kernel answers
  // Closure index of every (innermost direct class, userset class tgc) pair of the two-level steps (kernels.cuh
  // ClosureRef; built by gpu_build_closure, unsharded engines only). A pair over the size budget has none.
  struct Closure {
    uint16_t inner = 0, tgc = 0;
    DevBuf row_ptr, col;
    uint32_t nsubj = 0;
    uint64_t entries = 0;
    uint8_t width = 0;   // bytes per entry, 2 or 4: one width for every pair of the snapshot (build_closures)
    bool done = false;   // the budget was checked against this snapshot's relationships
    bool built = false;  // ... and the index built
    // Signature of every row (kernels.cuh sig_word / sig_mask): sig_words 64-bit words per row, row-major. 0: none (the
    // pair's steps meet through closure_meet).
    DevBuf sig;
    uint32_t sig_words = 0;
    double sig_ms = 0;  // device time of its last build
    // Set table of every row (closure_sig.cuh table_bucket; 16-bit indexes whose target type holds fewer than 65 536
    // objects): set_hdr one header word per row, set_tab set_buckets buckets of four 16-bit slots. Empty when
    // !set_built (the pair's steps meet through sig_meet or closure_meet).
    DevBuf set_hdr, set_tab;
    uint64_t set_buckets = 0;
    bool set_built = false;
    double set_ms = 0;  // device time of its last build
  };
  std::vector<Closure> closure;
  // Range records (kernels.cuh FlatRecordRef; gpu_build_flat_records) of the class gc of every push step of an SF_FLAT
  // slot: object obj's row is row_ptr[row_base + obj * ncls], obj < nres. Rebuilt whole by every publish that may change
  // the class's rows (finish_publish, and publish_delta when the journal touches gc). Empty when !built (over budget,
  // or a failed build): its steps then read the CSR.
  struct FlatRecords {
    uint16_t gc = 0;
    uint64_t row_base = 0;
    uint32_t nres = 0, ncls = 0;
    DevBuf rec;
    bool built = false;
    uint64_t long_rows = 0;  // rows longer than a record holds, read from the CSR
    double ms = 0;           // device time of its last build
  };
  std::vector<FlatRecords> records;
  uint64_t n_tuples = 0, bytes = 0, revision = 0;
  ~Snapshot();
};

// Device mirror of the interned names (ingress.cuh), built on the first device-ingress call and synced at the start
// of every one: the arena bytes past `bytes` are uploaded, their records inserted into the table, and the table is
// rebuilt at twice the size when its load would pass 1/2.
struct IngressMirror {
  struct Type {
    DevBuf arena, offs, slots;
    std::vector<uint64_t> host_offs;  // record offsets, as uploaded to offs
    uint64_t bytes = 0;               // arena bytes mirrored
    uint64_t cap = 0;                 // table slots (power of two), 0 = no table yet
  };
  std::vector<Type> types;
  // staging of zg_check_bulk_packed_ingress (offsets and blobs, pinned host -> device; items; answers) and the
  // resolve's scratch (the one subject's bytes, the decreasing-offset flag)
  DevBuf stage, items, out, one, bad;
  void *pin = nullptr, *pin_out = nullptr;
  size_t pin_cap = 0, pin_out_cap = 0;
  uint64_t names = 0, sync_uploads = 0, rebuilds = 0, items_resolved = 0;
  ~IngressMirror();
  uint64_t device_bytes() const;
};

// Sharded handle: where a level's queries go. Queries are written straight into their owners' inboxes (peer memory),
// and values are read back where their owners left them. p[d] = shard d's buffer, base[d] = where this shard's part of
// it starts. Passed to the kernels by value.
constexpr int kMaxShards = 64;  // = kMaxRouteDest (kernels.cuh)
struct PeerTable {
  void* p[kMaxShards];
  unsigned long long base[kMaxShards];
};

// A prefix filter's bitmaps (Device::prefix_scan): per type, ids whose interned name has the prefix.
struct PrefixBits {
  std::vector<const uint32_t*> type;  // per type: its bitmap, nullptr when the filter cannot select the type
  std::vector<uint32_t> n_ids;        // per type: the ids it covers (the snapshot's object capacity)
  uint64_t bytes = 0;                 // device bytes of the bitmaps
};
struct PrefixStats {
  uint64_t names = 0, matched = 0, launches = 0, syncs = 0;  // records scanned, ids set, launches, syncs that uploaded
};

class Device {
 public:
  ~Device();
  std::string init(int device, uint64_t subq_cap, uint32_t budget);
  std::string publish(const HostSnapshot& h, const Schema& sc, uint64_t revision);  // host-built arrays
  // Builds the CSR on the GPU (build.cu); verify: also build on the host and compare every array.
  std::string publish_gpu(const Store& store, const Schema& sc, uint64_t revision, bool verify);
  // Merges the store's journal into the resident snapshot. Returns "" on success, "full" when only a rebuild
  // can publish this state (no snapshot, re-layout, bulk load, huge delta), else an error message.
  std::string publish_delta(const Store& store, const Schema& sc, uint64_t revision);
  uint64_t delta_publishes = 0, full_publishes = 0;
  uint64_t closure_builds = 0;    // closure indexes built (the rebuilds after writes included)
  uint64_t closure_failures = 0;  // builds that failed (the pair met through batch_l2 until its next build)
  double closure_ms = 0;          // device time of the closure index builds of the last publish
  // ZGPU_VERIFY_BUILD=1: every array of the resident snapshot against the host builder's
  std::string verify_against_host(const Store& store, const Schema& sc);
  std::string verify_snapshot(Snapshot& s, const Store& store, const Schema& sc, const HostSnapshot* lay);
  double last_build_ms = 0;

  // d_items / d_out are device pointers. count_bytes != nullptr selects the
  // instrumented kernel variant. Returns ZG_* and fills err.
  int check_device(const zg_check* d_items, uint64_t n, uint8_t* d_out, cudaStream_t st, bool raw_items,
                   uint64_t* count_bytes, std::string* err, bool top = true, const unsigned long long* ready = nullptr);
  int check_host(const zg_check* items, uint64_t n, uint8_t* out, std::string* err);
  // Several callers' requests answered by ONE launch sequence (see Batcher in capi.cu).
  struct HostReq {
    const zg_check* items;
    uint64_t n;
    uint8_t* out;
  };
  int check_host_multi(const std::vector<HostReq>& reqs, std::string* err);
  int lookup(uint16_t res_type, const zg_check& proto, std::vector<uint32_t>* ids, std::string* err);
  // K <= 64 LookupResources in one launch sequence (multi-source reverse walk, one verification launch, one
  // sort, one copy back). rcs[i] = ZG_OK / ZG_EDEPTH per lookup; the call's own code covers the batch.
  struct LookupReq {
    uint16_t res_type;
    zg_check proto;
  };
  int lookup_batch(const std::vector<LookupReq>& reqs, std::vector<std::vector<uint32_t>>* ids, std::vector<int>* rcs,
                   std::string* err);
  uint64_t lookup_batches = 0, lookups_batched = 0;
  // One page of LookupResources: the first `want` answers with id > after (every id when !has_after), ascending, in
  // *ids. The candidates are those of lookup() (the reverse walk, the exhaustive list, the flat union), plus `self`
  // (ZG_NO_OBJECT: none), the userset subject's own object. Those after the cursor are sorted once, then verified in
  // windows from the front, each larger than the last, until `want` answers are found or the candidates run out.
  // ZG_EDEPTH when a candidate at or before the last answer found (the end, when fewer than `want` follow) cannot be
  // decided.
  struct LookupPageStats {
    uint64_t after = 0;     // candidates after the cursor (a repeat of the flat union counts per row)
    uint64_t verified = 0;  // candidates run through the check kernel
    uint64_t windows = 0;   // verification windows
  };
  int lookup_page(uint16_t res_type, const zg_check& proto, bool has_after, uint32_t after, uint64_t want, uint32_t self,
                  std::vector<uint32_t>* ids, LookupPageStats* st, std::string* err);
  // LookupSubjects (T:res#perm, subjects of type stype[#srel]): forward walk from the resource (else every object of
  // stype when the walk overflows or use_rbfs is off), the wildcard probe, one verification launch, a second
  // one without wildcard relationships when the wildcard is granted, compaction, sort, one copy back. ids:
  // subjects listed concretely, ascending; excluded: subjects the granted wildcard does not cover (only with
  // include_wildcard). ZG_EDEPTH when the probe or a candidate cannot be decided.
  struct SubjectsAnswer {
    std::vector<uint32_t> ids, excluded;
    bool wildcard = false;       // the wildcard entry is present
    bool fell_back = false;      // every object of the subject type was verified
    uint64_t n_verified = 0;     // items of the first verification launch (probe included)
  };
  int lookup_subjects(uint16_t res_type, uint32_t res, uint16_t perm, uint16_t stype, uint16_t srel, bool include_wildcard,
                      SubjectsAnswer* ans, std::string* err);
  uint64_t subject_lookups_walk = 0, subject_lookups_exhaustive = 0, subject_items_verified = 0;

  // ---- object-hash sharded store: one pass at a time, everything resident on the device (dist.DeviceShardedChecker) ----
  uint32_t shard_count = 1, shard_rank = 0;
  // Bucketises n check items by owner = res % n_dest into d_routed (destination-major) with their source
  // indices in d_src; counts[d] (host) = items for destination d. d_items == nullptr: the sub-queries raised by
  // pass `level` (shard_pass_dev).
  int route_by_owner(const zg_check* d_items, uint64_t n, int level, uint32_t n_dest, zg_check* d_routed, uint32_t* d_src,
                     uint64_t* counts, std::string* err);
  // Evaluates `n` device queries as pass `level` (level 0: caller items routed to this shard; deeper: routed
  // sub-queries, depth in flags). *n_sub = sub-queries this pass raised.
  int shard_pass_dev(const zg_check* d_queries, uint64_t n, int level, uint64_t* n_sub, std::string* err);
  // d_child_vals: one byte per raised sub-query in ROUTED order, d_src = the source indices route_by_owner wrote.
  // d_out: one byte per query of the level (v1 codes when final_codes, else value bits).
  int shard_fold_dev(int level, const uint8_t* d_child_vals, const uint32_t* d_src, uint64_t n_sub, uint8_t* d_out,
                     bool final_codes, std::string* err);
  int unroute(const uint32_t* d_src, const uint8_t* d_val, uint64_t n, uint8_t* d_out, std::string* err);
  // ---- LookupResources on the sharded store (dist.DeviceShardedLookup): one round of K <= 64 lookups at a time ----
  // Starts a round (the same lookups on every rank; home[k] = rank that asked lookup k) and clears its visited slices.
  // d_seeds receives the K level-0 frontier entries; walk_cap bounds every frontier and the walk's candidates.
  int shard_lookup_begin(const std::vector<LookupReq>& reqs, const uint8_t* home, uint64_t walk_cap,
                         unsigned long long* d_seeds, std::string* err);
  // Expands the n_in entries of d_front (level `level` of the replicated frontier) against this shard's reverse rows
  // into d_next (walk_cap entries). *overflow: the frontier or the candidates did not fit.
  int shard_lookup_expand(const unsigned long long* d_front, uint64_t n_in, int level, unsigned long long* d_next,
                          uint64_t* n_next, bool* overflow, std::string* err);
  // The round's candidates on this shard as check items: the walk's (exhaustive: every owned resource of the type)
  // plus the self-membership of owned userset subjects. d_items == nullptr: *n = the capacity d_items needs.
  int shard_lookup_candidates(bool exhaustive, zg_check* d_items, uint64_t cap, uint64_t* n, std::string* err);
  // Codes of the candidates -> answer keys (lookup << 32 | id; undecidable ones flagged) in d_routed, bucketed by home
  // rank; counts[d] (host) = keys for rank d.
  int shard_lookup_route(const uint8_t* d_codes, uint64_t n, uint32_t n_dest, unsigned long long* d_routed, uint64_t* counts,
                         std::string* err);
  // Keys that arrived home -> d_ids, ascending per lookup in lookup order; per_lookup[k] (host, K) = answers of
  // lookup k; *err_mask bit k: lookup k had an undecidable candidate.
  int shard_lookup_finish(const unsigned long long* d_keys, uint64_t n, uint32_t* d_ids, uint64_t* per_lookup,
                          uint64_t* err_mask, std::string* err);
  // ---- one shard of a sharded handle (zg_config.n_shards, capi.cu run_sharded): the handle drives every shard --------
  // The handle's ONE store holds every shard's relationships; this device's snapshot keeps those whose resource id %
  // own_count == own_rank (shard_rank / shard_count equal them). own_count = 1: the store is this device's alone.
  uint32_t own_rank = 0, own_count = 1;
  // Level 0: copies in this shard's n callers' items (pinned host or this device's memory) and counts them by owner:
  // counts[d] (host, own_count). Waits for the counts (a round trip).
  int peer_begin(const zg_check* items, uint64_t n, uint64_t* counts, std::string* err);
  // The inbox of `level` on this shard, grown to n queries; the level then holds n queries.
  zg_check* peer_inbox(int level, uint64_t n, std::string* err);
  // Writes the queries of `level` this shard sends (level 0: its callers' items; deeper: what pass level - 1 raised)
  // into the owners' inboxes at t.p[d] + t.base[d] + ..., and where each went; then records peer_event(level).
  int peer_scatter(int level, const PeerTable& t, std::string* err);
  // After every shard's peer_event(level) (`wait`, one per shard): evaluates the level's queries in one pass and counts
  // the sub-queries it raised by owner: *n_sub, counts[d] (host). Waits for them (a round trip). ZG_ENOMEM with
  // *overflow: the pass raised more than the sub-query capacity; the batch must be answered in halves. no_wildcards:
  // the pass runs with KParams::no_wildcards (LookupSubjects' second verification, on every pass of every shard).
  int peer_pass(int level, const std::vector<cudaEvent_t>& wait, uint64_t* n_sub, uint64_t* counts, bool* overflow,
                bool no_wildcards, std::string* err);
  // When pass `level` raised sub-queries: after every shard's peer_event(level + 1), ORs their values (t.p[d] = shard
  // d's values of level + 1) into the raising leaves and folds the level; records peer_event(level).
  int peer_fold(int level, const PeerTable& t, const std::vector<cudaEvent_t>& wait, std::string* err);
  const uint8_t* peer_values(int level) const { return pl_[static_cast<size_t>(level)].out.as<uint8_t>(); }
  // After every shard's peer_event(0): the answers of this shard's callers' items (t as in peer_fold, level 0) -> out
  // (pinned host or this device's memory). Waits for them (a round trip).
  int peer_finish(const PeerTable& t, const std::vector<cudaEvent_t>& wait, uint8_t* out, std::string* err);
  cudaEvent_t peer_event(int level) const { return ev_peer_[level & 1]; }  // alternates: a fold waits on one, records the other
  // LookupResources on a sharded handle (capi.cu run_sharded_lookup drives the shard_lookup_* round above on every
  // shard): the walk's buffers of this shard. front[level & 1] = the replicated frontier `level` expands, next = what
  // this shard's expand found (walk capacity), items / codes = its candidates and their codes, routed = its answer
  // keys, keys / ids = every shard's keys and the answers (shard 0). LookupSubjects on the handle (run_sharded_subjects)
  // uses front[0] as this shard's frontier, inbox for the walk entries the shards deliver to it, and items / codes /
  // routed / keys / ids as above. Both rounds run under the handle's device lock, so they never interleave.
  struct HandleLookupBufs {
    DevBuf front[2], next, items, codes, routed, keys, ids, inbox;
  } hl;
  bool hl_ensure(DevBuf& b, uint64_t bytes);  // b (one of hl) grown to bytes on this device
  uint64_t lookup_walk_cap() const { return lb_cap_; }
  // Writes n 8-byte entries of src (this device) to t.p[d] + t.base[d] for every d < n_dest, then records
  // peer_event(level). Runs on this shard's stream: its next work cannot overwrite src before they are written.
  int peer_put(const unsigned long long* src, uint64_t n, uint32_t n_dest, const PeerTable& t, int level, std::string* err);
  // This shard's next work starts after `wait` (other shards' peer_event of a level), with no host wait.
  int peer_wait(const std::vector<cudaEvent_t>& wait, std::string* err);
  // shard_pass_dev with KParams::no_wildcards (LookupSubjects' second verification, on every pass of every rank)
  int shard_pass_nowild_dev(const zg_check* d_queries, uint64_t n, int level, uint64_t* n_sub, std::string* err);
  // ---- LookupSubjects on the sharded store (dist.DeviceShardedLookup.lookup_subjects): one round of K <= 64 ----
  struct SubjectsReq {  // T:res#perm, subjects of type stype[#srel]
    uint32_t res;
    uint16_t res_type, perm, stype, srel;
  };
  // A round ends a LookupResources round begun on the same engine, and the other way round: they share buffers.
  // Starts a round (the same lookups on every rank; home[k] = rank that asked lookup k; include bit k: lookup k
  // asks for the wildcard entry). The owner of each written resource admits it as the level-0 frontier (d_front,
  // walk_cap entries; *n_front) and holds the lookup's probe item (and, with the walk, the resource as a candidate
  // when it has the subject type).
  int shard_subjects_begin(const std::vector<SubjectsReq>& reqs, const uint8_t* home, uint64_t include, uint64_t walk_cap,
                           unsigned long long* d_front, uint64_t* n_front, std::string* err);
  // Expands this rank's frontier (n_in entries of one level) over its forward rows; the discoveries, bucketed by
  // owner, go to d_routed (walk_cap entries); counts[d] (host) = entries for rank d. *overflow: an outbox, a frontier
  // or the candidates of the round did not fit (sticky for the round); nothing is routed then.
  int shard_subjects_expand(const unsigned long long* d_front, uint64_t n_in, uint32_t n_dest, unsigned long long* d_routed,
                            uint64_t* counts, bool* overflow, std::string* err);
  // The sharded handle's expand (capi.cu run_sharded_subjects): expands this shard's frontier into its outbox and counts
  // the outbox by owner on the device (the outbox size read there), with one wait for the flags and counts[d] (host,
  // shard_count), where shard_subjects_expand waits and then routes into a local buffer. *overflow as there; the
  // counts are then zero. The outbox stays put for shard_subjects_scatter.
  int shard_subjects_expand_count(const unsigned long long* d_front, uint64_t n_in, uint64_t* counts, bool* overflow,
                                  std::string* err);
  // Writes the n entries of the outbox into their owners' inboxes at t.p[d] + t.base[d] + ... (peer memory), then
  // records peer_event(level). No wait.
  int shard_subjects_scatter(uint64_t n, const PeerTable& t, int level, std::string* err);
  // Admits the n_in entries that arrived from every rank: the fresh ones are the next frontier (d_next, walk_cap).
  int shard_subjects_admit(const unsigned long long* d_in, uint64_t n_in, unsigned long long* d_next, uint64_t* n_next,
                           std::string* err);
  // This rank's candidates as check items: the probes, then the walk's candidates (exhaustive: every owned id of the
  // subject type). d_items == nullptr: *n = the capacity d_items needs.
  int shard_subjects_candidates(bool exhaustive, zg_check* d_items, uint64_t cap, uint64_t* n, std::string* err);
  // Codes of the first verification -> this rank's part of the round's granted / failed masks (host).
  int shard_subjects_verdicts(const uint8_t* d_codes, uint64_t n, uint64_t* granted, uint64_t* failed, std::string* err);
  // With the masks of every rank OR-ed: the answer keys of the first verification are kept, and the HAS candidates
  // of granted lookups go to d_items (cap >= the candidates) for the no-wildcards verification; *n_nw of them.
  int shard_subjects_nowild(const uint8_t* d_codes, uint64_t n, uint64_t granted, uint64_t failed, zg_check* d_items, uint64_t cap,
                            uint64_t* n_nw, std::string* err);
  // Codes of the no-wildcards verification: its HAS subjects are listed; every key goes to d_routed, bucketed by home
  // rank; counts[d] (host) = keys for rank d.
  int shard_subjects_route(const uint8_t* d_codes, uint64_t n, uint32_t n_dest, unsigned long long* d_routed, uint64_t* counts,
                           std::string* err);
  // Keys that arrived home -> d_ids: the listed ids of lookup 0, 1, ... then the excluded ids of lookup 0, 1, ...,
  // ascending each; listed[k] / excluded[k] (host, K) = their counts. Ends the round.
  int shard_subjects_finish(const unsigned long long* d_keys, uint64_t n, uint32_t* d_ids, uint64_t* listed, uint64_t* excluded,
                            std::string* err);

  // ---- relationship filters (filter.cuh): ReadRelationships, DeleteRelationships, write preconditions ----
  enum FilterShape { kByResource = 0, kBySubject = 1, kByScan = 2 };
  static FilterShape filter_shape(const Store::Filter& f) {
    return f.has_res ? kByResource : (f.has_subj || f.subj_wildcard) ? kBySubject : kByScan;
  }
  // The relationships of the resident snapshot that match f at clock `now` (0: expired ones too), what Store::match
  // returns for the store the snapshot was published from: *count of them, and with `tuples` the records, in no
  // particular order (expires, optional, parallel to them). A count launch sizes the output, then an emit launch fills
  // it. *too_big: the records would take more than a quarter of the free device memory; only *count is valid.
  // px: the filter's prefix bitmaps (prefix_scan; nullptr when the filter has no prefix), whose bytes count against
  // that budget.
  int match_filter(const Schema& sc, const Store::Filter& f, uint32_t now, uint64_t* count, std::vector<zg_tuple>* tuples,
                   std::vector<uint32_t>* expires, bool* too_big, std::string* err, const PrefixBits* px = nullptr);
  // The relationships of the resident snapshot whose expiration is set and <= before (zg_collect_expired), what
  // Store::expired returns for the store the snapshot was published from; otherwise as match_filter. Only the classes
  // with CF_EXPIRY are read. A count launch that finds nothing is the whole call.
  int match_expired(const Schema& sc, uint32_t before, uint64_t* count, std::vector<zg_tuple>* tuples, bool* too_big,
                    std::string* err);
  // A page (zg_read_relationships_page): the first `want` relationships of the resident snapshot that match f at
  // clock `now` (0: expired ones too) and whose key follows *after (nullptr: from the start), in K order (PageKey),
  // with their expirations. The scan and resource shapes walk windows of one type's objects at a time (filter.cuh
  // page_walk), the subject shape takes `want` entries of every selected class's reverse row and merges them here.
  // *too_big: the output would take more than a quarter of the free device memory, or a type has more selected
  // classes than one plan holds; nothing else is valid and the caller pages on the host.
  // With a prefix (px), the scan shape's windows are sized over the ascending list of each type's matched ids
  // (filter.cuh prefix_list_kernel), which counts against the budget with the bitmaps.
  struct PageStats {
    uint64_t scanned = 0, launches = 0;  // entries the windows covered (see zg_page_counters), kernel launches
    uint64_t list_launches = 0;          // of those, the launches that built and searched the match lists
  };
  int page_filter(const Schema& sc, const Store::Filter& f, uint32_t now, const PageKey* after, uint64_t want,
                  std::vector<zg_tuple>* tuples, std::vector<uint32_t>* expires, PageStats* st, bool* too_big,
                  std::string* err, const PrefixBits* px = nullptr);
  // zg_retire_unused_names: per type, one bit per id of the snapshot's object capacity, set where a relationship of
  // the snapshot names the id as its resource or its subject (filter.cuh mention_scan_kernel); OR-ed into *bits
  // (Store::IdBits, grown to the capacities). One launch per 64 types, one copy back.
  int scan_mentions(const Schema& sc, Store::IdBits* bits, std::string* err);

  // ---- resource id prefixes (ingress.cuh prefix_match_kernel) ----
  // Brings the names mirror in step with the store (ingress_sync), then sets, per type the filter may select (res_type,
  // or every type with a relation when res_type < 0), one bit per id of the snapshot's object capacity whose name
  // starts with `prefix`: one launch per 64 types. The bitmaps live on this device until the next call; the shards of a
  // sharded handle read them through peer memory. *too_big: they would take more than a quarter of the free device
  // memory, or the names mirror could not be brought up to date for lack of device memory (the mirror is then
  // dropped); nothing else is valid and the caller answers on the host. The caller holds the device lock and the names lock (shared is enough).
  int prefix_scan(const Store& store, const Schema& sc, int res_type, const std::string& prefix, PrefixBits* out,
                  PrefixStats* st, bool* too_big, std::string* err);

  // ---- device ingress (ingress.cuh): packed string ids -> interned checks against the mirror of the store's names ----
  // The literal fields of a packed call, resolved once on the host exactly as zg_resolve_checks_packed resolves them.
  struct IngressLiterals {
    zg_check base;       // every item starts as this (ok == false: answers ZG_ITEM_ERROR)
    bool ok = false;
    int rt = -1, st = -1;  // resource / subject type
    uint32_t one_su = ZG_NO_OBJECT;  // the one subject's id (one_subj != nullptr)
    const char* one_subj = nullptr;  // HOST bytes of the one subject, or nullptr: per-item subjects
    size_t one_len = 0;
  };
  // Brings the mirror in step with the store's names (creating it on first use), then resolves the n packed items
  // (DEVICE blobs and n + 1 offsets) into d_out on `st` and waits for it. The caller holds the names lock, shared or
  // exclusive. ZG_EINVAL when an offset decreases.
  int ingress_resolve(const Store& store, const IngressLiterals& lit, const char* d_res_ids, const uint32_t* d_res_off,
                      const char* d_subj_ids, const uint32_t* d_subj_off, uint64_t n, zg_check* d_out, cudaStream_t st,
                      std::string* err);
  // HOST blobs and offsets -> v1 codes in out: staged through pinned memory, resolved and checked on the engine's
  // stream in one launch sequence. The offsets are checked on the host while they are staged.
  int ingress_check_host(const Store& store, const IngressLiterals& lit, const char* res_ids, const uint32_t* res_off,
                         const char* subj_ids, const uint32_t* subj_off, uint64_t n, uint8_t* out, std::string* err);
  void ingress_reset() { ingress_.reset(); }  // a schema (re)load: the names are gone
  std::unique_ptr<IngressMirror> ingress_;     // nullptr until the first device-ingress call

  // ---- ExpandPermissionTree (expand.cuh) ----
  struct ExpandReq {
    uint32_t res;   // ZG_NO_OBJECT or past the snapshot's objects: a never-written object
    uint32_t tmpl;    // the slot's template root (Schema::x_root)
    uint32_t ncount;  // its counted (relation leaf / arrow) nodes
  };
  // The trees of reqs, level by level: *nodes / *subjects as zg_expand_permission_trees returns them (the failed
  // requests' nodes compacted away), (*status)[i] = ZG_OK / ZG_EDEPTH. ZG_ENOMEM when the nodes plus subjects of the
  // call, with the next level's jobs and a level's (job, counted node) pairs, pass `cap`. The scratch is freed before
  // returning.
  int expand(const std::vector<ExpandReq>& reqs, uint64_t cap, std::vector<zg_expand_node>* nodes,
             std::vector<zg_expand_subject>* subjects, std::vector<int32_t>* status, std::string* err);
  uint64_t x_trees = 0, x_levels = 0, x_nodes_out = 0, x_subjects_out = 0;
  std::vector<double> x_last_ms;  // the last call: per level, count, scan and emit milliseconds (CUDA events)

  // ---- zg_import_relationships (import.cuh) ----
  // One group of an import, its literal fields resolved on the host (HOST blobs and offsets, as the caller passed them).
  struct ImportGroup {
    const char *res_ids, *subj_ids;
    const uint32_t *res_off, *subj_off;
    uint64_t item0, n;  // call position of its first item, its items
    uint32_t rtype, stype, rel, rel_index, srel;
    uint32_t pos_plain, pos_wild, k_plain, k_wild;  // class positions in K and class indexes (~0u: no such class)
  };
  struct ImportCheck {
    uint64_t bad = ~0ull, dup = ~0ull;  // smallest call positions of a malformed id / a duplicate
    uint64_t found = 0;                 // name occurrences the store had
    std::vector<uint64_t> new_keys;     // the new names, (type << 48 | first occurrence), sorted
    std::vector<uint64_t> new_hash;     // their hash_bytes, in that order
    std::vector<uint64_t> type_count;   // new names per type
    double ms_names = 0, ms_sort = 0, ms_dups = 0;  // device time of the steps
  };
  // Steps 1-4 of import.cuh for the n items of `groups` (syncing the name mirror first): new names, temporary ids, the
  // smallest positions of malformed ids and of duplicates in the call and, when `locate`, against this device's
  // resident snapshot. Changes nothing but the import's scratch. `extent`: every type's id extent (Store::extent).
  int import_check(const Store& store, const std::vector<ImportGroup>& groups, uint64_t n, const std::vector<uint32_t>& extent,
                   bool locate, ImportCheck* out, std::string* err);
  // A shard of a sharded handle: the duplicates against its own snapshot of the items `src` (the shard that ran
  // import_check, its scratch read through peer memory) holds, of the resources it owns; the smallest position in *dup.
  int import_locate(const Device& src, uint64_t* dup, std::string* err);
  // Step 5: the temporary ids to `ids` (per type, concatenated from base[type]), and the n tuples back in call order.
  int import_finish(const std::vector<uint32_t>& ids, const std::vector<uint64_t>& base, const std::vector<uint32_t>& rtype_of_rel,
                    std::vector<zg_tuple>* tuples, std::string* err);
  // Frees the import's scratch: an import is a rare load or resync call, and its scratch is several times its input.
  void import_release();
  struct ImportScratch;
  struct ImportScratchFree {  // defined in device.cu, where ImportScratch is complete
    void operator()(ImportScratch* x) const;
  };
  std::unique_ptr<ImportScratch, ImportScratchFree> import_;

  std::shared_ptr<Snapshot> snap;
  cudaStream_t stream = nullptr;
  int device = 0;
  uint64_t launches = 0, passes = 0, checks = 0;
  uint64_t coalesced_launches = 0, coalesced_requests = 0;
  uint64_t streamed_calls = 0;  // host calls whose items were streamed in behind the running kernel
  uint64_t split_batches = 0;  // batches answered in halves because their sub-queries overflowed the pass buffer
  // cumulative device-side event counters: stack spills to HBM, batches that switched the path memo on
  void read_events(uint64_t* spills, uint64_t* memo_batches);
  int read_phase_clocks(uint64_t* cycles, std::string* err);  // ZG_PHASE_CLOCKS builds: 5 cumulative phase totals
  uint64_t lookups_rbfs = 0, lookups_exhaustive = 0, lookups_flat = 0;
  bool use_rbfs = true;  // ZGPU_NO_RBFS=1: LookupResources checks every resource of the type  // batcher: launches that served > 1 caller
  double last_ms = 0;
  bool invert = true;  // direction-optimised probes (ZG_FLAG_FORWARD_ONLY / ZGPU_NO_INVERT=1 disable)
  uint32_t now = 0;  // clock for expiration, set by the caller before each hot-path call
  uint64_t last_alg_bytes = 0;
  // Checks of flat_check_kernel's passes left to check_kernel so far: a synchronous device read, ordered after the
  // last check call's kernels on whatever stream they were enqueued (zg_stats_get)
  uint64_t flat_residual();

 private:
  uint64_t closure_cap_ = ~0ull;  // ZGPU_CLOSURE_CAP: entries a closure index may hold (tests; ~0 = the size budget)
  uint32_t closure_sig_words_ = ~0u;  // ZGPU_CLOSURE_SIG_WORDS: signature words per row (tests; 0 = none, ~0 = chosen
                                      // from the mean row length, gpu_build_closure_sig)
  bool closure_table_ = true;  // ZGPU_CLOSURE_TABLE: build the rows' set tables (tests; 0 = none)
  bool flat_check_ = true;     // ZGPU_FLAT_CHECK: mark SF_FLAT slots at publish (tests and A/B runs; 0 = none)
  bool flat_records_ = true;   // ZGPU_FLAT_RECORDS: build the SF_FLAT push steps' range records (tests and A/B; 0 = none)
  // (Re)builds the closure index of every pair of s->closure that is not built yet (`rebuild` false) or whose inner or
  // tgc class is marked in `rebuild` (a write changed it), from the classes' reverse rows described by h.cls. Decides
  // the entry width from h's object capacities first: 16-bit when every pair's tgc resource type holds at most 65 536
  // objects, else 32-bit, and rebuilds every pair built at another width. A pair whose build fails is left without an
  // index (closure_failures). Every index built here gets its signatures; a pair whose signatures fail keeps its index.
  void build_closures(Snapshot* s, const HostSnapshot& h, const std::vector<uint8_t>* rebuild);
  // (Re)builds the range records of s->records whose class is marked in `rebuild` (every one when null). A build that
  // fails leaves the class without records.
  void build_flat_records(Snapshot* s, const std::vector<uint8_t>* rebuild);
  // match_filter / match_expired: the count launch over the classes `sel` (p holds the rest of the plan), then with
  // `tuples` the emit launch sized by it, of filter_expired_kernel (`expired`) or the kernel of `shape`.
  int run_filter(const Schema& sc, const Snapshot& s, const std::vector<FilterSel>& sel, FilterPlan& p, FilterShape shape,
                 bool expired, uint64_t* count, std::vector<zg_tuple>* tuples, std::vector<uint32_t>* expires, bool* too_big,
                 std::string* err, const std::vector<const uint32_t*>* bits = nullptr, uint64_t held = 0);
  int ingress_sync(const Store& store, cudaStream_t st, std::string* err);
  std::string finish_publish(std::shared_ptr<Snapshot> s, const HostSnapshot& lay, const Schema& sc, uint64_t revision);
  // One check_kernel launch over `nq` queries: val (may be null) receives the per-(query, leaf) value
  // bits, out (may be null) the per-query v1 codes / value bits. lean: the queries are callers' (level 0 of an
  // unsharded engine): when the snapshot has SF_FLAT slots and meets through set tables, flat_check_kernel answers
  // theirs first and check_kernel only the rest.
  int run_pass(const Snapshot& s, const zg_check* queries, uint64_t nq, uint8_t* val, uint8_t* out, bool final_codes,
               bool raw, zg_check* subq, uint32_t* subq_parent, cudaStream_t st, bool count, std::string* err,
               const unsigned long long* ready = nullptr, bool lean = false);
  int sm_count_ = 0, blocks_per_sm_ = 0, blocks_per_sm_count_ = 0;
  uint32_t spill_cap_ = 4096, budget_ = 1u << 20;
  uint64_t subq_cap_ = 1ull << 22;
  DevBuf spill_, ctrl_, memo_;
  DevBuf flat_ctrl_, flat_idx_;  // flat_check_kernel: [0] the pass's residual, [1] the running total; the residual list
  uint32_t memo_entries_ = 8192, memo_after_ = 2048;  // ctrl: [0] next, [1] subq_count, [2] alg_bytes, then flags u32;
                                                      // [8 .. 9] events, [10] items landed, [11 .. 15] phase clocks
  std::vector<DevBuf> q_, parent_, val_;  // per pass level: queries, raising (query, leaf), leaf values
  std::vector<uint64_t> shard_nq_, shard_nsub_;  // sharded mode: queries / raised sub-queries per level
  DevBuf route_ctrl_;
  DevBuf stage_in_, stage_out_, lk_jobs_, lk_codes_, lk_ids_;
  DevBuf rb_visited_, rb_front_[2], rb_cand_;
  DevBuf lb_params_, lb_owner_, lb_ctrl_, lb_keys_[2];  // batched lookups
  DevBuf lp_sel_, lp_sorted_, lp_out_, lp_ctrl_;        // lookup pages: selected and sorted candidates, answers, control
  uint64_t lp_first_ = 1024;  // lookup pages: the first window's floor (ZGPU_LOOKUP_PAGE_WINDOW)
  uint32_t lp_growth_ = 4;    // and the least factor a window grows by (ZGPU_LOOKUP_PAGE_GROWTH)
  DevBuf ls_jobs_, ls_codes_, ls_has_, ls_ids_, ls_ctrl_;   // LookupSubjects
  DevBuf flt_out_, flt_exp_, flt_ctrl_;                     // match_filter: records, expirations, the count
  DevBuf pg_count_, pg_off_, pg_tmp_, pg_seg_;              // page_filter: tile counts, offsets, scan space, segments
  DevBuf mention_bits_;                                     // scan_mentions: every type's bitmap
  DevBuf px_bits_, px_str_, px_ctrl_;                       // prefix_scan: bitmaps, the prefix's bytes, the match count
  DevBuf px_first_, px_ids_, px_ent_, px_sum_, px_tmp_;     // prefix pages: a type's match list and its entry sums
  // sharded LookupResources round: walk state in rb_visited_ / lk_jobs_ / lb_owner_ / lb_params_ / lb_keys_ (a sharded
  // engine never runs lookup_batch), the round's home ranks, self-membership list and control words here
  DevBuf sl_home_, sl_self_, sl_ctrl_;
  std::shared_ptr<Snapshot> sl_snap_;  // the round reads one snapshot from begin to finish (released there)
  std::vector<LookupReq> sl_reqs_;
  uint64_t sl_cap_ = 0, sl_n_cand_ = 0;
  uint64_t sl_n_walk_ = 0;  // candidates before the self-membership ones: only these can fail a lookup
  // sharded LookupSubjects round: visited slices, candidates, params and keys in the buffers above; the outbox,
  // the no-wildcards items, home ranks and control words here
  DevBuf ss_out_, ss_nw_, ss_nw_owner_, ss_home_, ss_ctrl_;
  std::shared_ptr<Snapshot> ss_snap_;  // read from begin to finish (released there)
  std::vector<SubjectsReq> ss_reqs_;
  std::vector<zg_check> ss_probes_;  // this rank's probe items (the lookups whose resource it owns) and their lookups
  std::vector<uint8_t> ss_probe_owner_;
  uint64_t ss_cap_ = 0, ss_include_ = 0, ss_n_cand_ = 0, ss_n_nw_ = 0;
  template <bool kSrc, class Item, class Owner>
  int route_(const Item* d_items, uint64_t n, uint32_t n_dest, Owner owner, Item* d_routed, uint32_t* d_src, uint64_t* counts,
             std::string* err);
  // sharded handle: per level, the queries the shards delivered here, their leaf values and values, and the sub-queries
  // the pass raised (their raising (query, leaf), where their owners put them); the callers' items of level 0 in home_
  struct PeerLevel {
    DevBuf in, val, out, raised, parent, pos;
    uint64_t nq = 0, nsub = 0;
  };
  std::vector<PeerLevel> pl_;
  DevBuf home_, home_pos_, home_out_, peer_ctrl_;  // peer_ctrl_: counts[64], cursors[64]
  uint64_t home_n_ = 0;
  unsigned long long* pin_peer_ = nullptr;  // pinned: the control words and counts a round trip reads
  cudaEvent_t ev_peer_[2] = {nullptr, nullptr};
  int peer_events_(std::string* err);  // creates ev_peer_ on first use
  bool no_wildcards_ = false;  // run_pass: KParams::no_wildcards (LookupSubjects' second verification)
  uint64_t lb_cap_ = 1ull << 24;  // frontier entries / candidates of one lookup batch (ZGPU_LOOKUP_BATCH_CAP)
  void* pin_lk_ = nullptr;
  size_t pin_lk_cap_ = 0;
  uint64_t rb_cap_ = 1ull << 22;  // frontier / candidate capacity before falling back to the exhaustive scan
  // Reverse-BFS candidates of type res_type for the subject in proto; *overflow -> use the exhaustive list.
  int lookup_candidates(const Snapshot& s, uint16_t res_type, const zg_check& proto, uint64_t* n_cand, bool* overflow,
                        std::string* err);
  // streamed admission (check_host_multi): copy stream, "reset done" event, pinned per-chunk counters
  cudaStream_t cstream_ = nullptr;
  cudaEvent_t ev_reset_ = nullptr;
  unsigned long long* pin_ready_ = nullptr;
  size_t pin_ready_cap_ = 0;
  static constexpr uint64_t kStreamChunkItems = 1ull << 17;  // 2 MB of items per chunk
  static constexpr uint64_t kStreamMinItems = 1ull << 18;    // smaller calls: one plain copy
  static constexpr uint64_t kParallelGatherItems = 1ull << 20;  // coalesced groups from here on are gathered by helpers
  static constexpr unsigned kGatherThreads = 8;
  void* pin_in_ = nullptr;
  void* pin_out_ = nullptr;
  size_t pin_in_cap_ = 0, pin_out_cap_ = 0;
  cudaEvent_t ev0_ = nullptr, ev1_ = nullptr, last_done_ = nullptr;
  bool have_last_ = false;
  bool timing_pending_ = false;

 public:
  void finish_timing();
};

// Build time and tuning macros of the kernels in this library.
const char* build_info();

// Device radix sort of n u32 keys (build.cu keeps the cub instantiations in one translation unit).
std::string sort_u32(const uint32_t* d_in, uint32_t* d_out, uint64_t n, cudaStream_t st);
std::string sort_u64(const unsigned long long* d_in, unsigned long long* d_out, uint64_t n, int end_bit, cudaStream_t st);
// Owner filter (rank, count) of both: only the relationships whose resource id % count == rank (Store::build).
std::string gpu_build_snapshot(const Store& store, const Schema& sc, HostSnapshot* lay, cudaStream_t st, Snapshot* s,
                               uint32_t owner_rank = 0, uint32_t owner_count = 1);
// Applies store.journal to the arrays of `s` (same layout). cls_delta: per-class change of the relationship count.
// "relayout" / "corrupt": the caller must rebuild.
std::string gpu_apply_delta(const Store& store, const Schema& sc, const HostSnapshot& lay, cudaStream_t st, Snapshot* s,
                            std::vector<uint32_t>* cls_delta, uint32_t owner_rank = 0, uint32_t owner_count = 1);
// (Re)builds s->resources[] / n_resources[] from the forward row table.
std::string gpu_resource_lists(Snapshot* s, cudaStream_t st);
// Size budget of a closure index: entries (before duplicates are removed) per relationship of its two classes. cfg3's
// shape (8 memberships per user, 10 teams per group) needs about 9.
constexpr uint64_t kClosureRatio = 16;
// Builds the closure index of the pair (a, b) from the resident reverse CSR of s into *c with entries of c->width bytes
// (2 only when every resource id of class b is below 65 536), unless it would hold more than cap entries (~0: the
// budget above) or more than a quarter of the free device memory; c->built tells which.
std::string gpu_build_closure(const Snapshot& s, const DCls& a, const DCls& b, uint64_t cap, Snapshot::Closure* c,
                              cudaStream_t st);
// Builds the signatures of the built closure index *c: `words` 64-bit words per row (a power of two, 1 .. 32), or, with
// words = ~0u, the fewest with 64 * words >= 12 x the mean row length (about 1 % false "maybe"s per test at 3 bits per
// entry). None (c->sig_words = 0) when they would take more than a quarter of the free device memory.
std::string gpu_build_closure_sig(Snapshot::Closure* c, uint32_t words, cudaStream_t st);
// Builds the set table of the built 16-bit closure index *c (closure_sig.cuh), trying `seeds` seeds per bucket count.
// None (c->set_built false) when the index is 32-bit, a row would need more than kTableMaxBuckets buckets, or the table
// would take more than a quarter of the free device memory. The caller builds it only for a target type of fewer than
// 65 536 objects (0xFFFF marks an empty slot).
std::string gpu_build_closure_table(Snapshot::Closure* c, uint32_t seeds, cudaStream_t st);
// Builds the range records *r of one class from the resident forward CSR of s (kernels.cuh FlatRecordRef). None
// (r->built false) when they would take more than a quarter of the free device memory. The caller builds them only
// for a class whose subjects' type holds fewer than 65 536 objects.
std::string gpu_build_flat_records(const Snapshot& s, Snapshot::FlatRecords* r, cudaStream_t st);

}  // namespace zg
