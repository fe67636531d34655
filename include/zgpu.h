/*
 * zgpu.h -- C ABI of libzgpu.so: an H100-native (sm_90a) batched Zanzibar
 * permission-check engine that drops in behind the reference proxy's
 * v1.PermissionsServiceClient boundary (authzed/spicedb-kubeapi-proxy,
 * pkg/proxy/options.go:81-82,371-377).
 *
 * Every entry point is what a cgo shim implementing v1.PermissionsServiceClient
 * would bind (INTEGRATION.md shows that shim). Plain pointers and sizes only; the
 * caller owns every buffer, the library copies what it keeps and never retains a
 * caller pointer past return; nothing throws or aborts across this boundary.
 *
 * Reference interface each group replaces (file:line in /root/reference):
 *   zg_check_bulk*              CheckBulkPermissions   pkg/authz/check.go:41-69,
 *                                                      pkg/authz/postfilter.go:127-178
 *                               CheckPermission        pkg/authz/watch.go:50-67
 *   zg_lookup_resources*        LookupResources stream pkg/authz/lookups.go:49-88
 *   zg_lookup_subjects*         LookupSubjects stream  (v1 API; pkg/authz/postfilter_test.go:71 mock)
 *   zg_write_relationships      WriteRelationships     pkg/authz/distributedtx/activity.go:54-76
 *   zg_delete_relationships     DeleteRelationships    (v1 API; filter semantics update.go:207-271)
 *   zg_collect_expired          the datastore's garbage collection of expired relationships (pkg/spicedb/spicedb.go:53)
 *   zg_retire_unused_names      frees the interned names no relationship mentions any more, for reuse
 *   zg_read_relationships       ReadRelationships      pkg/authz/distributedtx/activity.go:128-171
 *   zg_read_relationships_page  ReadRelationships with optional_limit / optional_cursor (v1 API)
 *   zg_delete_relationships_limited  DeleteRelationships with optional_limit / optional_allow_partial_deletions
 *   zg_watch_read               WatchService.Watch     pkg/authz/watch.go:27-48
 *   zg_engine_create/load_schema embedded SpiceDB ctor pkg/spicedb/spicedb.go:18-57
 *
 * Return codes: 0 = OK, negative = error (message: zg_last_error).
 */
#ifndef ZGPU_H
#define ZGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ZG_OK 0
#define ZG_EINVAL (-1)   /* bad argument / schema violation                      */
#define ZG_EEXIST (-2)   /* CREATE of an existing relationship                   */
#define ZG_ENOSCHEMA (-3)
#define ZG_ECUDA (-4)    /* CUDA error: the call fails closed                     */
#define ZG_EPRECOND (-5) /* a WriteRelationships precondition did not hold       */
#define ZG_ENOSNAPSHOT (-6) /* nothing published yet                             */
#define ZG_E2BIG (-7)    /* output buffer too small; required size reported      */
#define ZG_ENOMEM (-8)
#define ZG_EDEPTH (-9)   /* LookupResources / LookupSubjects: a candidate hit the dispatch-depth cap / work budget */

/* v1.CheckPermissionResponse.Permissionship (authzed-go v1.6.0); per-item codes */
#define ZG_NO_PERMISSION 1
#define ZG_HAS_PERMISSION 2
#define ZG_CONDITIONAL 3 /* never produced: caveats are out of scope              */
#define ZG_ITEM_ERROR 255 /* per-item error (depth > 50, unknown permission ...)  */

#define ZG_SREL_NONE 0xFFFFu     /* subject has no relation ("" or "...")          */
#define ZG_SREL_WILDCARD 0xFFFEu /* stored relationship whose subject is type:*   */
#define ZG_NO_OBJECT 0xFFFFFFFFu /* object id of a name that was never written    */

#define ZG_OP_TOUCH 0  /* v1.RelationshipUpdate_OPERATION_TOUCH  */
#define ZG_OP_CREATE 1 /* v1.RelationshipUpdate_OPERATION_CREATE */
#define ZG_OP_DELETE 2 /* v1.RelationshipUpdate_OPERATION_DELETE */

#define ZG_PRECOND_MUST_MATCH 1     /* v1.Precondition_OPERATION_MUST_MATCH     */
#define ZG_PRECOND_MUST_NOT_MATCH 2 /* v1.Precondition_OPERATION_MUST_NOT_MATCH */

#define ZG_MAX_DEPTH 50 /* pkg/spicedb/spicedb.go:33 WithDispatchMaxDepth(50) */

typedef struct zg_engine zg_engine;

/* zg_config.flags: build schema/store/snapshot on the host only (CPU unit tests of
 * the host logic). Every hot-path call on such an engine FAILS with ZG_ECUDA:
 * there is no CPU evaluation path in this library. */
#define ZG_FLAG_HOST_ONLY 1u
/* Forward expansion only: every direct probe is a binary search of the resource's row
 * (no direction-optimised probes from the subject's reverse rows). For A/B measurement. */
#define ZG_FLAG_FORWARD_ONLY 2u
/* Sharded handle (n_shards > 1) only: the handle answers zg_lookup_resources, zg_lookup_resources_str and
 * zg_list_prefilter itself. Each round's reverse walk runs on every shard, its frontier and answer keys exchanged
 * through peer memory, and its candidates are verified by the handle's check protocol (zg_handle_lookup_counters).
 * The answers equal a replica's. On any other engine, zg_engine_create returns ZG_EINVAL. */
#define ZG_FLAG_HANDLE_LOOKUPS 4u
/* Sharded handle (n_shards > 1) only, independent of ZG_FLAG_HANDLE_LOOKUPS: the handle answers zg_lookup_subjects and
 * zg_lookup_subjects_str itself, one lookup per call. Its forward walk runs on every shard, each discovery written into
 * its owner's inbox through peer memory; the candidates are verified by the handle's check protocol, the second
 * (no-wildcards) verification too (zg_handle_subjects_counters). The answers equal a replica's. On any other engine,
 * zg_engine_create returns ZG_EINVAL. */
#define ZG_FLAG_HANDLE_SUBJECTS 8u

typedef struct {
  int32_t device;            /* CUDA device ordinal; -1 = current device          */
  uint32_t flags;            /* ZG_FLAG_*                                         */
  uint64_t subquery_capacity; /* 0 = default; sub-queries buffered per pass       */
  uint32_t work_budget;      /* 0 = default; expansion rounds per 32-check batch
                                before unresolved checks report ZG_ITEM_ERROR
                                (the analogue of a request deadline)              */
  uint16_t shard_rank;       /* object-hash sharded store: this engine keeps only    */
  uint16_t shard_count;      /* relationships whose resource id % count == rank;
                                0 or 1 = whole store (replica)                       */
  uint32_t n_devices;        /* 0 / 1 = the one device above; k > 1 = devices device .. device + k - 1, each
                                holding a replica of the snapshot and answering its slice of every bulk call
                                (SURVEY.md 8e mode 1: no data-path collective); ZG_ALL_DEVICES = every
                                visible device from `device` on                                            */
  uint32_t n_shards;         /* 0 / 1 = one store per device (above); S > 1 = this ONE handle holds the S shards of an
                                object-hash sharded store: shard k keeps the relationships whose resource id % S == k
                                and lives on device `device + k % D` (D = n_devices, 1 by default; with one GPU the
                                S shards share it). Checks cross the shards in-process, sub-queries delivered through
                                peer memory; every device pair must have peer access. Not with shard_count > 1;
                                S <= 64. LookupResources / LookupSubjects / the list pre-filter, zg_check_bulk_device,
                                the device-ingress calls and the zg_shard_*_dev calls are refused (ZG_EINVAL);
                                with ZG_FLAG_HANDLE_LOOKUPS, LookupResources and the list pre-filter are answered,
                                with ZG_FLAG_HANDLE_SUBJECTS, LookupSubjects. */
} zg_config;
#define ZG_ALL_DEVICES 0xFFFFFFFFu

/* One interned check: 16 bytes in, 1 byte out. Object ids are dense per type. */
typedef struct {
  uint32_t res;   /* resource object id (type implied by perm)                    */
  uint32_t subj;  /* subject object id                                            */
  uint16_t perm;  /* slot id of the permission OR relation being checked          */
  uint16_t stype; /* subject type id                                              */
  uint16_t srel;  /* subject relation slot id, or ZG_SREL_NONE                    */
  uint16_t flags; /* 0                                                            */
} zg_check;

/* One interned relationship (pkg/rules/rules.go:1050 grammar, interned). */
typedef struct {
  uint32_t res;
  uint32_t subj;  /* ignored when srel == ZG_SREL_WILDCARD                        */
  uint16_t rel;   /* slot id of the relation (implies resource type)              */
  uint16_t stype;
  uint16_t srel;  /* slot id, ZG_SREL_NONE or ZG_SREL_WILDCARD                    */
  uint16_t flags; /* 0                                                            */
} zg_tuple;

typedef struct {
  zg_tuple t;
  uint32_t expires_at; /* unix seconds, 0 = never (OptionalExpiresAt)             */
  uint32_t op;         /* ZG_OP_*                                                 */
} zg_update;

/* String forms: what the Go shim passes straight from the v1 protobuf messages. */
typedef struct {
  const char *res_type, *res_id, *relation; /* relation or permission name        */
  const char *subj_type, *subj_id, *subj_rel; /* subj_rel NULL/""/"..." = none     */
} zg_rel_str;

typedef struct {
  zg_rel_str rel;
  uint32_t expires_at;
  uint32_t op;
} zg_update_str;

/* v1.RelationshipFilter (pkg/authz/update.go:207-271): NULL/"" = unset field.   */
typedef struct {
  const char *res_type, *res_id, *relation;
  const char *subj_type, *subj_id, *subj_rel;
} zg_filter_str;

typedef struct {
  uint32_t op; /* ZG_PRECOND_* */
  zg_filter_str filter;
} zg_precondition_str;

typedef struct {
  uint64_t checks;          /* checks answered since creation                     */
  uint64_t launches;        /* kernels launched since creation                    */
  uint64_t passes;          /* sub-query passes beyond the first                  */
  uint64_t tuples;          /* relationships in the published snapshot            */
  uint64_t snapshot_bytes;  /* device bytes of the published snapshot             */
  uint64_t revision;        /* increments on every publish                        */
  uint64_t last_alg_bytes;  /* algorithmic bytes of the last counted call         */
  double last_kernel_ms;    /* device time of the last hot-path call              */
  uint64_t coalesced_launches; /* launches that answered more than one concurrent caller */
  uint64_t coalesced_requests; /* zg_check_bulk calls answered by those launches         */
  uint64_t stack_spills;       /* warp stacks that overflowed shared memory into HBM     */
  uint64_t memo_batches;       /* 32-check batches that switched the path memo on        */
  uint64_t split_batches;      /* batches answered in halves (sub-query buffer overflow) */
  uint64_t delta_publishes;    /* publishes that merged a journal of updates into the resident snapshot */
  uint64_t full_publishes;     /* publishes that rebuilt the snapshot from the relationship list        */
  double last_publish_ms;      /* device time of the last publish (merge or rebuild)                    */
  uint64_t streamed_calls;     /* host calls whose items were copied in behind the running kernel       */
  uint64_t lookup_batches;     /* launch sequences that answered more than one LookupResources           */
  uint64_t lookups_batched;    /* LookupResources calls answered by those                                */
  uint64_t devices;            /* GPUs this engine owns (counters above are summed over them)            */
  uint64_t shards;             /* zg_config.n_shards of a sharded handle, else 1                         */
  uint64_t last_levels;        /* sharded handle, last coalesced group: pass levels run over the shards  */
  uint64_t last_subqueries;    /*   sub-queries the shards raised to each other                          */
  uint64_t last_round_trips;   /*   times the host waited for the devices                                */
  uint64_t flat_slots;         /* slots of the published program whose checks the lean flat-check kernel */
                               /*   answers (SF_FLAT; 0 when ZGPU_FLAT_CHECK=0)                          */
  uint64_t flat_residual;      /* checks of those kernel's batches it left to the check kernel, in all   */
} zg_stats;

/* ---- lifecycle --------------------------------------------------------- */
int zg_engine_create(const zg_config *cfg, zg_engine **out);
void zg_engine_destroy(zg_engine *e);
/* Message of the last failing call ON THE CALLING THREAD (thread-local, so concurrent callers never see
 * each other's text). A caller whose runtime migrates it between OS threads from one foreign call to the
 * next (Go) must fetch it on the thread of the failing call: pin the goroutine around the pair
 * (runtime.LockOSThread; go/gpuauthz/client.go `call`) or wrap call + zg_last_error_copy in one C
 * function of the cgo preamble. zg_last_error_copy writes at most cap - 1 bytes + NUL into buf and
 * returns the full length of the message. */
const char *zg_last_error(void);
size_t zg_last_error_copy(char *buf, size_t cap);

/* ---- schema (SpiceDB schema DSL subset; pkg/spicedb/bootstrap.yaml) ----- */
int zg_load_schema(zg_engine *e, const char *dsl, size_t len);
int zg_num_types(const zg_engine *e);
int zg_num_slots(const zg_engine *e);
int zg_type_id(const zg_engine *e, const char *type_name);            /* -1 unknown */
int zg_slot_id(const zg_engine *e, int type_id, const char *name);    /* -1 unknown */
int zg_slot_type(const zg_engine *e, int slot);
int zg_slot_is_permission(const zg_engine *e, int slot);
const char *zg_slot_name(const zg_engine *e, int slot);
const char *zg_type_name(const zg_engine *e, int type_id);

/* ---- object interning (string id <-> dense per-type u32) ---------------- */
uint32_t zg_intern_object(zg_engine *e, int type_id, const char *object_id);
uint32_t zg_find_object(const zg_engine *e, int type_id, const char *object_id); /* ZG_NO_OBJECT */
/* Copies the name into buf (NUL terminated); returns its length or ZG_E2BIG/ZG_EINVAL. */
int zg_object_name(const zg_engine *e, int type_id, uint32_t id, char *buf, size_t cap);
/* Bulk zg_intern_object over the packed layout: the n ids are [off[i], off[i+1]) of ids. out_ids[i] = the id of
 * name i (an existing name keeps its id; the empty id gives ZG_NO_OBJECT, as zg_intern_object refuses it).
 * ZG_EINVAL for an unknown type or a decreasing offset (nothing is interned then). Host only. */
int zg_intern_objects_packed(zg_engine *e, int type_id, const char *ids, const uint32_t *off, uint64_t n,
                             uint32_t *out_ids);

/* ---- relationship store -------------------------------------------------- */
/* Bulk TOUCH of interned relationships (expires may be NULL). Not visible to
 * checks until zg_publish. */
int zg_load_tuples(zg_engine *e, const zg_tuple *t, const uint32_t *expires, uint64_t n);
/* Transactional CREATE/TOUCH/DELETE; all-or-nothing. Not visible until publish. */
int zg_apply_updates(zg_engine *e, const zg_update *u, uint64_t n);
/* Builds the CSR snapshot in HBM and makes it the one every later check sees. */
int zg_publish(zg_engine *e);
/* Drops every relationship (interned names and ids stay) and publishes the empty store: what a caller
 * that mirrors another source of truth does before re-loading it (go/gpuauthz resync). The watch feed
 * restarts at the new revision. */
int zg_clear_relationships(zg_engine *e);
uint64_t zg_num_tuples(const zg_engine *e);
/* Clock used for expiration; 0 = wall clock (default). */
void zg_set_clock(zg_engine *e, int64_t unix_seconds);

/* v1 WriteRelationships: validate, check preconditions, apply, publish. The
 * write is visible to every check that starts after return (FullyConsistent). */
int zg_write_relationships(zg_engine *e, const zg_update_str *updates, uint64_t n,
                           const zg_precondition_str *pre, uint64_t n_pre);
/* v1 ImportBulkRelationships: every relationship is a CREATE, and the call is all-or-nothing. Relationships come
 * in groups of one class, packed as zg_check_bulk_packed takes them. */
typedef struct {
  const char *res_type, *relation, *subj_type, *subj_rel; /* one class; subj_rel NULL or "" = none */
  const char *res_ids;                                    /* blob of resource ids */
  const uint32_t *res_off;                                /* n + 1 offsets into res_ids */
  const char *subj_ids;                                   /* blob of subject ids; "*" = the wildcard subject */
  const uint32_t *subj_off;                               /* n + 1 offsets into subj_ids */
  const uint32_t *expires_at;                             /* n, or NULL; 0 = no expiration */
  uint64_t n;
} zg_import_group;
/* Imports the groups' relationships in call order (groups in order, items in order) and publishes once.
 *   - Each relationship gets the checks zg_write_relationships makes of a CREATE. One that is already stored (an
 *     expired one not yet collected included), or that appears earlier in the call, fails with ZG_EEXIST. The error
 *     is that of the first failing relationship in call order: the code and message the write path gives for it,
 *     prefixed "relationship <call position> (<text>): ". On failure nothing changes: no name is interned, nothing
 *     is stored, the revision does not move and the watch feed gets no entry.
 *   - New names get the ids the same relationships would get written in the same order through
 *     zg_write_relationships: first appearance, the subject's name before the resource's; freed ids lowest first.
 *   - Pending changes are published with the import; the revision advances by one. Every relationship is recorded in
 *     the watch feed as a CREATE; an import larger than the feed holds clears it, and the feed restarts at the new
 *     revision as after zg_clear_relationships.
 *   - Names are resolved and interned, and duplicates found, on the GPU (the environment variable
 *     ZGPU_IMPORT_HOST=1 selects the host path); host-only engines run the host path. A sharded handle imports into
 *     its one store and rebuilds every shard. ZG_EINVAL on a standalone shard (zg_config.shard_count > 1): it cannot
 *     see the other shards' relationships.
 *   - At most 2^30 relationships per call (ZG_EINVAL above). The device scratch is freed when the call returns.
 *   - Takes the device lock, then the names lock exclusively, as a write does. *n_imported may be NULL. */
int zg_import_relationships(zg_engine *e, const zg_import_group *groups, uint64_t n_groups, uint64_t *n_imported);
/* out[0..4] = successful imports run on the device, on the host, relationships imported, name occurrences found
 * already interned, names interned new. */
int zg_import_counters(zg_engine *e, uint64_t *out);
/* The last successful import's steps, in milliseconds: ms[0..6] = names, sort and duplicates (device events; 0 on
 * the host path), the host's checks and interning, the store and its index, the publish, the whole call. */
int zg_import_last_times(zg_engine *e, double *ms);
/* v1 DeleteRelationships by filter; *n_deleted may be NULL. */
int zg_delete_relationships(zg_engine *e, const zg_filter_str *filter,
                            const zg_precondition_str *pre, uint64_t n_pre, uint64_t *n_deleted);
/* Removes every relationship whose expiration is set and <= before_unix from the store and from the resident
 * snapshot(s). before_unix must not be later than the engine's clock (zg_set_clock, else wall clock): ZG_EINVAL.
 * Every check, lookup and read at a clock >= before_unix answers as before the call. *n_removed may be NULL.
 *   - Relationships without an expiration (expires == 0) are never removed; a schema without expiration removes
 *     nothing. Nothing calls this automatically: a deployment runs it on its own schedule (INTEGRATION.md).
 *   - Takes the device lock, then the names lock exclusively, as zg_delete_relationships does.
 *   - When nothing qualifies it returns 0 removed: nothing is applied or published, the revision does not move. On a
 *     current snapshot that costs one count launch. Otherwise the DELETEs are applied and published once (pending
 *     changes included, as every write call does), and the revision advances.
 *   - It writes nothing to the watch feed: an expiration is not a write, and no answer at a clock >= before_unix
 *     changes. Interned names are kept, as after every delete.
 *   - Found on the device (a scan of the classes that may carry an expiration; every shard of a sharded handle scans
 *     its own rows) when the snapshot is current, else by a scan of the host store; zg_filter_counters counts it as
 *     it counts a delete by filter. */
int zg_collect_expired(zg_engine *e, int64_t before_unix, uint64_t *n_removed);
/* Retires every interned name (type, id) that no relationship in the store names as its resource or its subject (live,
 * expired and not yet collected, or loaded / applied and not yet published) and no change retained in the watch feed
 * names; *n_retired (may be NULL) = how many. Ids that bulk loads use without a name are never touched.
 *   - After the call a retired name is as if it had never been written: zg_find_object gives ZG_NO_OBJECT,
 *     zg_object_name of its old id ZG_EINVAL, and every string-form call answers as before, since nothing mentioned it.
 *     Names that are not retired keep their ids.
 *   - Nothing is published, the revision does not move, the watch feed records nothing, the snapshot is not touched.
 *   - Id reuse: later interning (zg_intern_object, zg_intern_objects_packed, the write calls) hands out the freed ids
 *     lowest first before it extends the type's id space, so object capacities stay flat under churn. A freed id that
 *     zg_load_tuples / zg_apply_updates names directly is no longer free.
 *   - A caller must not use an id of a retired name obtained earlier: until it is reused it answers as a never-written
 *     object, after reuse it denotes the new name. An engine on which this is never called behaves as before.
 *   - The lookup answers kept for the ZG_E2BIG protocol stay valid: every id in an answer is mentioned at its revision.
 *   - The string calls that resolve names and answer after releasing the names lock (zg_check_bulk_str,
 *     zg_check_bulk_packed, zg_lookup_resources_str, zg_lookup_subjects_str, zg_list_postfilter, zg_list_prefilter)
 *     resolve and answer again when a retirement ran in between, so they never answer for, or print, a name that
 *     took over a retired name's id. Each retirement that retires a name makes such calls in flight start over.
 *   - Takes the device lock, then the names lock exclusively, as zg_collect_expired does. ZG_EINVAL on a standalone
 *     shard (zg_config.shard_count > 1: its store does not hold the other shards' relationships); sharded handles and
 *     replicas are served. The device mirror of the names (device ingress) is dropped when a name is retired and
 *     rebuilt by the next device-ingress call.
 *   - The mentioned ids are read from the resident snapshot (every shard of a sharded handle scans its own, OR-ed)
 *     when it is the store, else by a scan of the host store (host-only engines, unpublished changes). */
int zg_retire_unused_names(zg_engine *e, uint64_t *n_retired);
/* Name counters (zg_stats keeps its layout): out[0] named objects, out[1] names retired since the schema was loaded,
 * out[2] free ids (retired, not reused yet), out[3] the id extent summed over types (the larger of the named and the
 * numeric ids: what object capacities follow), out[4] bytes of the host name arenas, out[5] / out[6] names retired by
 * calls that read the mentions on the device / by the host scan. */
int zg_name_counters(zg_engine *e, uint64_t *out);
/* The object capacity of type_id in the last layout (what the snapshot's row tables cover; 0 before the first
 * publish). Capacities grow in steps and never shrink; a capacity step makes the next publish a full rebuild. */
uint64_t zg_object_capacity(const zg_engine *e, int type_id);
/* Tests only: hook(arg) runs inside the string checks and lookups listed under zg_retire_unused_names, after they
 * resolved their names and before they answer, with no lock held (NULL removes it). */
int zg_debug_set_resolve_hook(zg_engine *e, void (*hook)(void *), void *arg);
/* v1 ReadRelationships: matching live relationships as "type:id#rel@stype:sid[#srel]\n"
 * lines, sorted. Returns 0 or ZG_E2BIG (*need = bytes required incl. NUL). */
int zg_read_relationships(zg_engine *e, const zg_filter_str *filter, char *buf, size_t cap,
                          size_t *need, uint64_t *n_out);

/* ---- pages of relationship reads, and deletes with a limit ---- */
/* A resumable position in a filter's matches (ReadRelationships' optional_cursor / after_result_cursor). Opaque, with
 * no public fields: it names the key of the last relationship returned, not a position, so it stays valid across
 * writes, collections, retirements and publishes. A cursor made for another filter, or before the schema was loaded
 * again, is refused with ZG_EINVAL. */
#define ZG_READ_CURSOR_BYTES 32
typedef struct zg_read_cursor {
  uint8_t opaque[ZG_READ_CURSOR_BYTES];
} zg_read_cursor;
/* One page of zg_read_relationships: the first `limit` (>= 1, else ZG_EINVAL) live relationships that match the filter
 * and follow `after` (NULL: from the start) in the page order. The page order is the key (resource type, resource id,
 * class position, subject id): the class position is the index of the relationship's (relation, subject type, subject
 * relation) among the classes of its resource type, in schema order. It depends on the schema and the interned ids
 * alone, so every engine kind (replicated, sharded handle, host only) and both paths give identical pages.
 *   - Lines use the text of zg_read_relationships, in the page order; expires[i] (NULL or *n_out entries) is line i's
 *     expiration (0 = none), cursors[i] (NULL or *n_out entries) the cursor that resumes after line i.
 *   - *next resumes after the page (after the last line; `after` itself, or the start, when the page is empty), *more
 *     is 1 exactly when another match follows the page.
 *   - A relationship that exists unchanged for the whole paging appears exactly once; one created or deleted between
 *     pages may appear or not.
 *   - ZG_E2BIG (*need = bytes required incl. NUL, *n_out = lines) fills nothing else: the caller's cursor still resumes
 *     where it did.
 *   - Locks and paths are those of zg_read_relationships: on a current snapshot the device answers (the first `limit` +
 *     1 matches after the cursor, in order, without visiting the rest of the store), otherwise the host store. A page
 *     never publishes. */
int zg_read_relationships_page(zg_engine *e, const zg_filter_str *filter, uint64_t limit, const zg_read_cursor *after,
                               char *buf, size_t cap, size_t *need, uint64_t *n_out, uint32_t *expires,
                               zg_read_cursor *cursors, zg_read_cursor *next, int32_t *more);
/* zg_delete_relationships with DeleteRelationships' optional_limit and optional_allow_partial_deletions. limit 0 is
 * zg_delete_relationships (*partial = 0). Otherwise, when more than `limit` relationships match (expired ones included,
 * as for zg_delete_relationships):
 *   - allow_partial == 0: ZG_EPRECOND, nothing changes;
 *   - allow_partial != 0: the first `limit` of them in the page order are deleted and *partial = 1
 *     (DELETION_PROGRESS_PARTIAL).
 * Else every match is deleted and *partial = 0 (DELETION_PROGRESS_COMPLETE). Preconditions, the watch feed and the
 * publish are those of zg_delete_relationships. *n_deleted and *partial may be NULL. */
int zg_delete_relationships_limited(zg_engine *e, const zg_filter_str *filter, const zg_precondition_str *pre,
                                    uint64_t n_pre, uint64_t limit, int allow_partial, uint64_t *n_deleted,
                                    int32_t *partial);
/* Cumulative counters of the pages of zg_read_relationships_page and zg_delete_relationships_limited: out[0] pages
 * served on the device, out[1] pages served by the host store, out[2] entries the device windows covered (forward
 * entries of the scanned objects; the resource shape: the row entries counted; the subject shape: the candidates read),
 * out[3] device launches. Pages also count in zg_filter_counters as filters. */
int zg_page_counters(zg_engine *e, uint64_t *out);

/* ---- filters by resource id prefix (v1.RelationshipFilter.optional_resource_id_prefix) ---- */
/* A zg_filter_str with a resource id prefix. res_id_prefix NULL or "" = unset: the filter is the zg_filter_str alone,
 * and every _ex call answers exactly as the call without _ex.
 *   - Match rule: a relationship matches when its resource has an interned name that starts with the prefix's bytes
 *     (byte-wise, case-sensitive). Ids that bulk loads use without a name never match, as they never match res_id.
 *     A retired name matches nothing; a reused id matches by its new name.
 *   - Validation: 1..1024 characters of [a-zA-Z0-9/_|\-=+] (`*` is not allowed), else ZG_EINVAL. res_id and the
 *     prefix together are ZG_EINVAL, as in SpiceDB.
 *   - The prefix needs no resource type: without one it selects matching resources of every type. (res_id and
 *     relation still need one.)
 *   - Everything else is as without the prefix: expiry at the engine's clock, deletes include expired relationships,
 *     limited deletes take the first `limit` in the page order, preconditions count matches, deletes write the watch
 *     feed and publish once.
 *   - A page cursor fingerprints the prefix when it is set: a cursor made with another prefix, or with none, is
 *     ZG_EINVAL. An unprefixed filter's cursors are those of zg_read_relationships_page.
 *   - On a current snapshot the device answers: it scans the device mirror of the interned names (the one device
 *     ingress keeps) for the matching resources, one bitmap per type, then runs the filter kernels against it. */
typedef struct {
  zg_filter_str f;
  const char *res_id_prefix; /* NULL/"" = unset */
} zg_filter_ex;
typedef struct {
  uint32_t op; /* ZG_PRECOND_* */
  zg_filter_ex filter;
} zg_precondition_ex;
int zg_read_relationships_ex(zg_engine *e, const zg_filter_ex *filter, char *buf, size_t cap, size_t *need,
                             uint64_t *n_out);
int zg_read_relationships_page_ex(zg_engine *e, const zg_filter_ex *filter, uint64_t limit, const zg_read_cursor *after,
                                  char *buf, size_t cap, size_t *need, uint64_t *n_out, uint32_t *expires,
                                  zg_read_cursor *cursors, zg_read_cursor *next, int32_t *more);
/* limit 0 = unlimited (zg_delete_relationships). */
int zg_delete_relationships_limited_ex(zg_engine *e, const zg_filter_ex *filter, const zg_precondition_ex *pre,
                                       uint64_t n_pre, uint64_t limit, int allow_partial, uint64_t *n_deleted,
                                       int32_t *partial);
int zg_write_relationships_ex(zg_engine *e, const zg_update_str *updates, uint64_t n, const zg_precondition_ex *pre,
                              uint64_t n_pre);
/* Cumulative counters of prefix filters (zg_filter_counters keeps its layout): out[0] prefix filters answered on the
 * device, out[1] prefix filters answered by the host store, out[2] names the device scanned, out[3] resources the
 * device matched, out[4] device launches of the prefix scans and their match lists, out[5] syncs of the names mirror
 * that uploaded bytes. */
int zg_prefix_counters(zg_engine *e, uint64_t *out);

/* ---- the hot path -------------------------------------------------------- */
/* CheckBulkPermissions: out[i] answers items[i] (same length, same order:
 * pkg/authz/check.go:54-57). HOST buffers; copies are inside the call. */
int zg_check_bulk(zg_engine *e, const zg_check *items, uint64_t n, uint8_t *out);
/* Same with DEVICE buffers on the given cudaStream_t (NULL = default stream);
 * asynchronous when the schema needs no sub-query pass. */
int zg_check_bulk_device(zg_engine *e, const zg_check *d_items, uint64_t n, uint8_t *d_out,
                         void *cuda_stream);
/* String form of CheckBulkPermissions / CheckPermission (n = 1): resolves, then takes the same
 * coalescing path as zg_check_bulk. */
int zg_check_bulk_str(zg_engine *e, const zg_rel_str *items, uint64_t n, uint8_t *out);
/* Only the resolution step of zg_check_bulk_str (strings -> interned checks; no GPU work, nothing is
 * interned: never-written names get the ZG_NO_OBJECT sentinels, unknown types / permissions give an
 * item that answers ZG_ITEM_ERROR). Lets a caller intern once and reuse the ids; they stay valid
 * until zg_retire_unused_names retires their name. */
int zg_resolve_checks(zg_engine *e, const zg_rel_str *items, uint64_t n, zg_check *out);
/* Packed form for a bulk request whose items share their literal fields (one rule template evaluated per
 * item: pkg/authz/postfilter.go:88-110): the n resource ids are the byte ranges
 * [res_off[i], res_off[i+1]) of res_ids (n + 1 offsets, no terminators); the subjects likewise, or with
 * subj_off == NULL ONE subject id for all items, NUL-terminated in subj_ids. Two buffers cross the
 * boundary instead of 6 n C strings. zg_check_bulk_packed = zg_resolve_checks_packed + zg_check_bulk. */
int zg_resolve_checks_packed(zg_engine *e, const char *res_type, const char *relation, const char *subj_type,
                             const char *subj_rel, const char *res_ids, const uint32_t *res_off,
                             const char *subj_ids, const uint32_t *subj_off, uint64_t n, zg_check *out);
int zg_check_bulk_packed(zg_engine *e, const char *res_type, const char *relation, const char *subj_type,
                         const char *subj_rel, const char *res_ids, const uint32_t *res_off,
                         const char *subj_ids, const uint32_t *subj_off, uint64_t n, uint8_t *out);
/* Device ingress: the same resolution on the GPU, against a device mirror of the interned names that the first such
 * call on an engine creates and every later one brings up to date (only names interned since are uploaded; a schema
 * load discards it). The items are bit-identical to zg_resolve_checks_packed's. Both calls take the device lock and
 * return after their GPU work has completed; they use the engine's first device.
 *   zg_resolve_checks_packed_device  DEVICE blobs, offsets and d_out, on cuda_stream (NULL = default stream). With
 *                                    d_subj_off NULL, d_subj_ids is the one subject as a HOST NUL-terminated string.
 *                                    ZG_EINVAL when an offset decreases. Allowed on sharded engines (it reads only
 *                                    names); composes with zg_check_bulk_device.
 *   zg_check_bulk_packed_ingress     zg_check_bulk_packed's arguments (HOST buffers): publishes pending writes, then
 *                                    stages the ids in pinned memory, resolves and checks them on the GPU and copies
 *                                    the answers back in one launch sequence. It does not join the coalescing batcher:
 *                                    small calls should keep using zg_check_bulk_packed. Refused on sharded engines.
 * ZG_ECUDA on host-only engines. */
int zg_resolve_checks_packed_device(zg_engine *e, const char *res_type, const char *relation, const char *subj_type,
                                    const char *subj_rel, const char *d_res_ids, const uint32_t *d_res_off,
                                    const char *d_subj_ids, const uint32_t *d_subj_off, uint64_t n, zg_check *d_out,
                                    void *cuda_stream);
int zg_check_bulk_packed_ingress(zg_engine *e, const char *res_type, const char *relation, const char *subj_type,
                                 const char *subj_rel, const char *res_ids, const uint32_t *res_off,
                                 const char *subj_ids, const uint32_t *subj_off, uint64_t n, uint8_t *out);
/* Cumulative device-ingress counters (zg_stats keeps its layout): out[0] names mirrored, out[1] device bytes of the
 * mirror, out[2] calls that uploaded names, out[3] table rebuilds (a full table re-inserted at twice the size),
 * out[4] items resolved on the device. All 0 before the first device-ingress call. */
int zg_ingress_counters(zg_engine *e, uint64_t *out);

/* LookupResources: ids (ascending) of every object of res_type with HAS_PERMISSION.
 * Returns 0, or ZG_E2BIG with *n_out = required capacity. */
int zg_lookup_resources(zg_engine *e, uint16_t res_type, uint16_t perm, uint16_t stype,
                        uint32_t subj, uint16_t srel, uint32_t *out_ids, uint64_t cap,
                        uint64_t *n_out);
/* String form: resource object ids as '\n'-separated lines. */
int zg_lookup_resources_str(zg_engine *e, const char *res_type, const char *perm,
                            const char *subj_type, const char *subj_id, const char *subj_rel,
                            char *buf, size_t cap, size_t *need, uint64_t *n_out);
/* Pages of LookupResources (optional_limit, optional_cursor, after_result_cursor). The order is ascending interned
 * resource id, the order zg_lookup_resources returns; it is not name order. A page is the first `limit` (>= 1, else
 * ZG_EINVAL) ids of the unpaged answer that follow `after` (NULL: from the start).
 *   - *more is 1 exactly when another answer follows the page. *next resumes after the page's last id (`after`
 *     itself, or the start, when the page is empty); cursors[i] (NULL or *n_out entries) resumes after id i.
 *   - The cursor is a zg_read_cursor under its own tag: it names the schema generation, the request (resource type,
 *     permission, subject type and relation, the subject as given: its id, or its name in the string form) and the
 *     last id. A read cursor, a cursor of another request or form, or one made before a schema load is ZG_EINVAL.
 *   - Pending writes are published first; the page is evaluated at the engine's clock. A cursor names an id, not a
 *     position: a resource that holds the permission for the whole paging appears exactly once, one that gains or
 *     loses it between pages may appear or not.
 *   - ZG_EDEPTH only when a candidate that cannot be decided lies after the cursor and at or before the page's
 *     deciding answer (the (limit + 1)-th, or the end when fewer follow). Where zg_lookup_resources succeeds, every page
 *     does; a page that ends before an undecidable resource succeeds where zg_lookup_resources fails. A sharded handle
 *     fails a page whenever the whole lookup has an undecidable candidate.
 *   - A replicated engine verifies only the candidates the page needs, in windows, on its first device. A sharded
 *     handle with ZG_FLAG_HANDLE_LOOKUPS runs the whole lookup and cuts the page from it (identical pages and cursors).
 *     Everything else is refused as zg_lookup_resources is (ZG_EINVAL; ZG_ECUDA on a host-only engine).
 * The string form renders at most `limit` names. A never-written userset subject that names itself (Check says so)
 * has no id: its name comes after every id, and its cursor is past the ids. ZG_E2BIG (*need = bytes incl. NUL, *n_out
 * = lines) fills nothing else, so the caller's cursor still resumes where it did; the retry runs the page again. */
int zg_lookup_resources_page(zg_engine *e, uint16_t res_type, uint16_t perm, uint16_t stype, uint32_t subj,
                             uint16_t srel, uint64_t limit, const zg_read_cursor *after, uint32_t *ids /* limit */,
                             uint64_t *n_out, zg_read_cursor *cursors, zg_read_cursor *next, int32_t *more);
int zg_lookup_resources_page_str(zg_engine *e, const char *res_type, const char *perm, const char *subj_type,
                                 const char *subj_id, const char *subj_rel, uint64_t limit,
                                 const zg_read_cursor *after, char *buf, size_t cap, size_t *need, uint64_t *n_out,
                                 zg_read_cursor *cursors, zg_read_cursor *next, int32_t *more);
/* Cumulative counters of LookupResources pages (zg_stats keeps its layout): out[0] pages answered by windowed
 * verification, out[1] pages cut from a whole answer (sharded handle), out[2] candidates after the cursor, out[3]
 * candidates verified, out[4] verification windows launched. */
int zg_lookup_page_counters(zg_engine *e, uint64_t *out);

/* LookupSubjects: which subjects of type stype[#srel] have `perm` on object `res` (of perm's type).
 * Subjects granted through their own relationships are listed in ids (ascending). When a wildcard
 * relationship (stype:*) grants perm and wildcard_option is ZG_WILDCARDS_INCLUDE, *wildcard = 1 and
 * `excluded` lists (ascending) the subjects the wildcard does not cover (`user:* - banned`); every
 * subject listed in neither has perm exactly when *wildcard is 1. With ZG_WILDCARDS_EXCLUDE the
 * wildcard entry is left out. Candidates come from a forward walk of the resident snapshot from res
 * (every object of stype when the walk overflows), verified by the check kernel. Returns 0; ZG_E2BIG
 * with *n_out / *n_excluded = required sizes; ZG_EDEPTH when a subject cannot be decided (depth cap /
 * work budget); ZG_EINVAL for unknown ids; ZG_ECUDA on a host-only engine. A sharded engine refuses this
 * call and the string form (ZG_EINVAL): use the zg_shard_subjects_*_dev calls (dist.DeviceShardedLookup). So does a
 * sharded handle (zg_config.n_shards > 1), unless it was created with ZG_FLAG_HANDLE_SUBJECTS: it then answers both
 * forms as a replica holding the same relationships does, the walk overflowing ZGPU_LOOKUP_BATCH_CAP straight into
 * verifying every object of the subject type. A resource id that no relationship names gives an empty answer. No
 * caveats, limits or cursors. */
#define ZG_WILDCARDS_INCLUDE 0u /* v1.LookupSubjectsRequest WILDCARD_OPTION_UNSPECIFIED / INCLUDE_WILDCARDS */
#define ZG_WILDCARDS_EXCLUDE 1u /* v1.LookupSubjectsRequest WILDCARD_OPTION_EXCLUDE_WILDCARDS               */
int zg_lookup_subjects(zg_engine *e, uint16_t perm, uint32_t res, uint16_t stype, uint16_t srel,
                       uint32_t wildcard_option, uint32_t *ids, uint64_t cap, uint64_t *n_out,
                       uint32_t *excluded, uint64_t ex_cap, uint64_t *n_excluded, int32_t *wildcard);
/* String form: '\n'-separated lines, one per concrete subject id; when the wildcard entry is present a
 * "*" line follows, then one "!<id>" line per excluded subject. *n_out = lines, *need = bytes incl. NUL. */
int zg_lookup_subjects_str(zg_engine *e, const char *res_type, const char *res_id, const char *perm,
                           const char *subj_type, const char *subj_rel, uint32_t wildcard_option,
                           char *buf, size_t cap, size_t *need, uint64_t *n_out);
/* Cumulative LookupSubjects counters of the engine's device (zg_stats keeps its layout): out[0] lookups answered
 * by the forward walk, out[1] lookups that verified every object of the subject type, out[2] check items of
 * their first verification launches (the probe included). */
int zg_lookup_subjects_counters(zg_engine *e, uint64_t *out);

/* ExpandPermissionTree (v1, shallow): the subject tree of object `res` (of perm's type, ZG_NO_OBJECT: a never-written
 * one) for relation or permission `perm`, built on the device from the resident forward CSR, one arrow level per
 * launch sequence (DESIGN.md §2 "ExpandPermissionTree" for the tree's shape). Pending writes are published first;
 * expired relationships are invisible at the engine's clock.
 *   - Every node has an expanded object (object, of `slot`'s type) and relation (`slot`) and is an intermediate node
 *     (ZG_EXPAND_UNION / INTERSECTION / EXCLUSION) or a leaf listing subjects[subjects, subjects + n_subjects): a
 *     relation's live relationships in class order, then ascending id, userset subjects not expanded further.
 *   - nodes[] holds the trees of the requests in order; a parent precedes its children, which rebuild the tree from
 *     (parent, rank). parent is UINT32_MAX for a root and otherwise an index into nodes[]; otherwise the order is the
 *     engine's, deterministic for one snapshot.
 *   - status[i]: ZG_OK, or ZG_EDEPTH when the tree would hold a subtree reached through more than ZG_MAX_DEPTH arrows
 *     (an arrow cycle); such a request contributes no node and the others are unaffected.
 * Returns ZG_OK; ZG_E2BIG with *n_nodes / *n_subjects = the required sizes (a retry computes the trees again);
 * ZG_EINVAL for an unknown slot, an id past the type's capacity, a slot whose tree template is too large, or a sharded
 * handle / standalone shard; ZG_ENOMEM when the call's nodes plus subjects, with the jobs of the next arrow level or
 * the (object, relation leaf or arrow) pairs of one level, pass the cap (ZGPU_EXPAND_CAP, default 2^26); ZG_ECUDA on a
 * host-only engine. A multi-device engine answers on its first device. */
#define ZG_EXPAND_UNION 1u /* v1 AlgebraicSubjectSet.Operation */
#define ZG_EXPAND_INTERSECTION 2u
#define ZG_EXPAND_EXCLUSION 3u
#define ZG_EXPAND_LEAF 4u
typedef struct {
  uint16_t perm;
  uint16_t pad;
  uint32_t res; /* may be ZG_NO_OBJECT */
} zg_expand_request;
typedef struct {
  uint32_t request, parent, rank; /* parent UINT32_MAX for a root; rank = position among the parent's children */
  uint32_t object;
  uint16_t slot, op;
  uint32_t n_subjects;
  uint64_t subjects; /* ZG_EXPAND_LEAF: its subjects[subjects, subjects + n_subjects) */
} zg_expand_node;
typedef struct {
  uint32_t id;
  uint16_t type, srel; /* srel: ZG_SREL_NONE, ZG_SREL_WILDCARD (id 0), or the userset's slot */
} zg_expand_subject;
int zg_expand_permission_trees(zg_engine *e, const zg_expand_request *reqs, uint64_t n, int32_t *status,
                               zg_expand_node *nodes, uint64_t node_cap, uint64_t *n_nodes,
                               zg_expand_subject *subjects, uint64_t subj_cap, uint64_t *n_subjects);
/* String form of one tree: one '\n'-terminated line per node in pre-order, children in rank order:
 * "<depth> <U|I|X|L> <type>:<id>#<relation>[ <subject>]*", depth = nesting depth (root 0), a subject written
 * type:id, type:id#rel or type:*. A never-written res_id gives the tree with empty leaves. *n_lines = nodes,
 * *need = bytes incl. NUL; ZG_E2BIG when cap is short; ZG_EDEPTH as status above; ZG_EINVAL for unknown names. */
int zg_expand_permission_tree_str(zg_engine *e, const char *res_type, const char *res_id, const char *perm, char *buf,
                                  size_t cap, size_t *need, uint64_t *n_lines);
/* Cumulative counters of the engine's first device: out[0] trees answered, out[1] levels launched, out[2] nodes,
 * out[3] subjects. */
int zg_expand_counters(zg_engine *e, uint64_t *out);
/* Device time of the last zg_expand_permission_trees call on the first device: per level, the count, scan and emit
 * milliseconds (CUDA events), 3 per level. *n = values; ZG_E2BIG when cap is short. */
int zg_expand_last_times(zg_engine *e, double *ms, uint64_t cap, uint64_t *n);
/* Cumulative LookupResources counters of a sharded handle with ZG_FLAG_HANDLE_LOOKUPS (zeros on any other engine):
 * out[0] rounds begun on the shards (a round answers up to 64 lookups; a halved round counts its halves too), out[1]
 * walk levels expanded, out[2] times the host waited for the shards (the verification's included), out[3] frontier
 * entries all-gathered, out[4] candidates verified, out[5] rounds redone in halves (a frontier or the candidates
 * overflowed ZGPU_LOOKUP_BATCH_CAP), out[6] rounds that verified every resource of the type (a single lookup that
 * overflowed, or ZGPU_NO_RBFS=1). */
int zg_handle_lookup_counters(zg_engine *e, uint64_t *out);
/* Cumulative LookupSubjects counters of a sharded handle with ZG_FLAG_HANDLE_SUBJECTS (zeros on any other engine):
 * out[0] lookups, out[1] walk levels expanded, out[2] times the host waited for the shards (both verifications'
 * included), out[3] walk entries written to another shard's inbox, out[4] candidates verified, out[5] items of the
 * no-wildcards verification, out[6] lookups that verified every object of the subject type (the walk overflowed
 * ZGPU_LOOKUP_BATCH_CAP, or ZGPU_NO_RBFS=1). */
int zg_handle_subjects_counters(zg_engine *e, uint64_t *out);
/* Cumulative counters of the relationship filters of zg_read_relationships, zg_delete_relationships and the
 * preconditions of both write calls (zg_stats keeps its layout). A filter is answered from the published snapshot on
 * the device when the engine has one and nothing was loaded or applied since; otherwise (host-only engines,
 * unpublished changes) by a scan of the host store. out[0] filters answered on the device, out[1] filters answered by
 * the host scan, out[2] relationships the device returned (a precondition only counts, and returns none), out[3..5]
 * device filters by shape: resource given, subject given without a resource, neither. */
int zg_filter_counters(zg_engine *e, uint64_t *out);
/* Closure indexes of the two-level steps in the engine's published snapshot (zg_stats keeps its layout): out[0] pairs
 * indexed, out[1] pairs over the size budget (their steps meet through the memberships' reverse rows instead), out[2]
 * index entries, out[3] index device bytes; out[4] index builds since creation (the rebuilds after writes included),
 * out[5] device microseconds of the last publish's index builds, out[6] builds that failed (that pair then meets
 * without an index until its next build). */
int zg_closure_index_counters(zg_engine *e, uint64_t *out);
/* Closure index `pair` (0-based, in the order of the program's two-level steps) of the published snapshot: out[0] 1 when
 * it is built, out[1] its entry width in bytes (2 when every id of its target type fits 16 bits, else 4; the same for
 * every pair of a snapshot), out[2] entries, out[3] device bytes. ZG_EINVAL when there is no such pair. */
int zg_closure_index_info(zg_engine *e, uint32_t pair, uint64_t *out);
/* Copies closure index `pair` (0-based, in the order of the program's two-level steps) of the published snapshot:
 * *n_rows + 1 row offsets to row_ptr, *n_entries entries to col (32-bit whatever the index's width). ZG_E2BIG (sizes
 * filled) when a buffer is too small, ZG_EINVAL when the pair has no index. For inspection and tests. */
int zg_closure_index_copy(zg_engine *e, uint32_t pair, uint32_t *row_ptr, uint64_t row_cap, uint32_t *col,
                          uint64_t col_cap, uint64_t *n_rows, uint64_t *n_entries);

/* Signatures of closure index `pair` (the check kernel tests a range's children against them and searches the row only
 * on a "maybe"): out[0] 1 when built, out[1] 64-bit words per row, out[2] bits set per entry, out[3] device bytes,
 * out[4] device microseconds of their last build. ZG_EINVAL when there is no such pair. */
int zg_closure_signature_info(zg_engine *e, uint32_t pair, uint64_t *out);
/* Copies the signatures of closure index `pair`, row-major (*n_words = rows x words per row). ZG_E2BIG (size filled)
 * when the buffer is too small, ZG_EINVAL when the pair has none. For inspection and tests. */
int zg_closure_signature_copy(zg_engine *e, uint32_t pair, uint64_t *words, uint64_t cap, uint64_t *n_words);

/* Set table of closure index `pair` (the check kernel looks a range's children up in it, exactly, instead of testing
 * signatures): out[0] 1 when built, out[1] buckets, out[2] 16-bit slots per bucket, out[3] device bytes (headers and
 * buckets), out[4] device microseconds of its last build. ZG_EINVAL when there is no such pair. */
int zg_closure_table_info(zg_engine *e, uint32_t pair, uint64_t *out);
/* Copies the set table of closure index `pair`: one header word per row (first bucket in bits 0-31, bucket count in
 * bits 32-55, seed in bits 56-63) and the buckets (four 16-bit slots each, 0xFFFF empty). ZG_E2BIG (sizes filled) when
 * a buffer is too small, ZG_EINVAL when the pair has none. For inspection and tests. */
int zg_closure_table_copy(zg_engine *e, uint32_t pair, uint64_t *hdr, uint64_t hdr_cap, uint64_t *buckets,
                          uint64_t bucket_cap, uint64_t *n_rows, uint64_t *n_buckets);

/* Range records `k` (the lean check kernel loads a range's children from them, by object, instead of through the
 * range's offsets): out[0] 1 when built, out[1] the edge class, out[2] objects, out[3] device bytes, out[4] rows longer
 * than a record holds (read through their offsets), out[5] device microseconds of their last build. ZG_EINVAL when
 * there are no such records. */
int zg_flat_record_info(zg_engine *e, uint32_t k, uint64_t *out);
/* Copies range records `k`: per object, one record of 16-bit slots (slot 0 the row's length, or 0xFFFF when it is too
 * long for the record; then the children in row order; 0xFFFF after them); *n_slots = objects x slots per record.
 * ZG_E2BIG (size filled) when the buffer is too small, ZG_EINVAL when there are none. For inspection and tests. */
int zg_flat_record_copy(zg_engine *e, uint32_t k, uint16_t *slots, uint64_t cap, uint64_t *n_slots);

/* Pinned host memory for request/response buffers: zg_check_bulk copies straight
 * from/to such buffers (no staging memcpy). */
void *zg_host_alloc(size_t bytes);
void zg_host_free(void *p);

/* Test hook: copies row (relation slot, resource id, edge class k) of the last
 * BUILT snapshot (host copy) into out; with bit 31 of cls set, the REVERSE row of that
 * class for subject id `res`. Returns 0 / ZG_E2BIG (*n_out = size). */
int zg_debug_row(zg_engine *e, uint16_t rel_slot, uint32_t res, uint32_t cls, uint32_t *out,
                 uint64_t cap, uint64_t *n_out);
/* The same row of shard `shard` of a sharded handle (zg_config.n_shards > 1): the host builder's arrays of the
 * relationships that shard owns. ZG_EINVAL on any other engine or shard index. */
int zg_debug_shard_row(zg_engine *e, uint32_t shard, uint16_t rel_slot, uint32_t res, uint32_t cls, uint32_t *out,
                       uint64_t cap, uint64_t *n_out);

/* ---- object-hash sharded store (one engine per GPU, shard_count > 1) --------
 * A check starts on the owner of its resource; an edge to an object owned by another shard (or
 * into a non-pure permission) is raised as a sub-query. The ranks run pass by pass and exchange
 * the raised sub-queries (all-to-all) until none are left, then fold the values back level by
 * level (spicedb-kubeapi-proxy_b200/dist.py DeviceShardedChecker). Every buffer stays resident on
 * the device: checks and raised sub-queries are bucketised by owner in a kernel, exchanged device to
 * device (NCCL all-to-all over NVLink, or peer copies), and the values coming back are folded without
 * a host copy. All pointers are DEVICE pointers of the engine's GPU; every call returns after its work
 * completed (the exchange runs on the caller's stream). On sharded engines zg_check_bulk /
 * zg_lookup_resources / zg_lookup_subjects are refused: use these zg_shard_*_dev calls (checks), the
 * zg_shard_lookup_*_dev calls below (LookupResources) or the zg_shard_subjects_*_dev calls (LookupSubjects).
 *   zg_shard_route_dev   items (d_items, or the sub-queries raised by pass `level` when d_items is NULL) ->
 *                        d_routed in destination-major order + d_src[i] = source index of d_routed[i];
 *                        counts[d] (HOST array of n_dest) = items for destination d = res % n_dest
 *   zg_shard_pass_dev    evaluates the level's n queries (d_queries) in one pass: level 0 takes the callers'
 *                        items routed to this shard, deeper levels the routed sub-queries with the hop depth in
 *                        flags; *n_sub = the sub-queries the pass raised
 *   zg_shard_fold_dev    d_child_vals in ROUTED order + the d_src of that routing -> d_out[q] per query of the
 *                        level (v1 codes when final_codes, else value bits for the rank that raised it)
 *   zg_shard_unroute_dev d_out[d_src[i]] = d_val[i]: answers restored to the caller's order */
int zg_shard_route_dev(zg_engine *e, const zg_check *d_items, uint64_t n, int level, uint32_t n_dest,
                       zg_check *d_routed, uint32_t *d_src, uint64_t *counts);
int zg_shard_pass_dev(zg_engine *e, const zg_check *d_queries, uint64_t n, int level, uint64_t *n_sub);
int zg_shard_fold_dev(zg_engine *e, int level, const uint8_t *d_child_vals, const uint32_t *d_src,
                      uint64_t n_sub, uint8_t *d_out, int final_codes);
int zg_shard_unroute_dev(zg_engine *e, const uint32_t *d_src, const uint8_t *d_val, uint64_t n, uint8_t *d_out);

/* LookupResources on a sharded engine (dist.DeviceShardedLookup), in rounds of k <= 64 lookups that every rank
 * runs with the same list. Shard r discovers, in its own reverse rows, only objects it owns, so the walk needs no
 * cross-shard dedup: each level every rank expands the whole replicated frontier and the next frontier is every
 * rank's new entries, all-gathered. Candidates are verified by the sharded check protocol above, and the answers are
 * sent to the rank that asked the lookup. Same conventions as the zg_shard_*_dev calls; ZG_EINVAL on an engine
 * that is not sharded, ZG_ECUDA on a host-only one. zg_lookup_resources* stays refused on sharded engines.
 *   zg_shard_lookup_begin_dev      starts a round: res_types / protos (subj, perm, stype, srel) / home (rank that
 *                                  asked) are HOST arrays of k; d_seeds (device, k entries) receives the level-0
 *                                  frontier; walk_cap bounds every frontier and the walk's candidates
 *   zg_shard_lookup_expand_dev     expands the n_in frontier entries of d_front against this shard's reverse rows
 *                                  into d_next (walk_cap entries): *n_next new entries; *overflow = 1 when a frontier
 *                                  or the candidates did not fit (redo the round in halves; a single lookup verifies
 *                                  every resource of its type instead)
 *   zg_shard_lookup_candidates_dev this shard's candidates as check items (the walk's, or with exhaustive every owned
 *                                  resource of the type, plus owned userset subjects naming their own object); with
 *                                  d_items NULL, *n = the capacity needed; ZG_E2BIG when cap is smaller
 *   zg_shard_lookup_route_dev      d_codes (one per candidate) -> answer keys (lookup << 32 | id; bit 38: a walk candidate
 *                                  could not be decided; an undecidable self-membership is left out, as in
 *                                  zg_lookup_resources) in d_routed, bucketed by home rank; counts[d] (HOST, n_dest)
 *   zg_shard_lookup_finish_dev     the keys that arrived home -> d_ids: ascending ids of lookup 0, then lookup 1, ...;
 *                                  per_lookup[i] (HOST, k) = ids of lookup i; *err_mask bit i: lookup i is ZG_EDEPTH */
int zg_shard_lookup_begin_dev(zg_engine *e, const uint16_t *res_types, const zg_check *protos, const uint8_t *home,
                              uint32_t k, uint64_t walk_cap, uint64_t *d_seeds);
int zg_shard_lookup_expand_dev(zg_engine *e, const uint64_t *d_front, uint64_t n_in, int level, uint64_t *d_next,
                               uint64_t *n_next, int *overflow);
int zg_shard_lookup_candidates_dev(zg_engine *e, int exhaustive, zg_check *d_items, uint64_t cap, uint64_t *n);
int zg_shard_lookup_route_dev(zg_engine *e, const uint8_t *d_codes, uint64_t n, uint32_t n_dest, uint64_t *d_routed,
                              uint64_t *counts);
int zg_shard_lookup_finish_dev(zg_engine *e, const uint64_t *d_keys, uint64_t n, uint32_t *d_ids, uint64_t *per_lookup,
                               uint64_t *err_mask);

/* LookupSubjects on a sharded engine (dist.DeviceShardedLookup.lookup_subjects), in rounds of k <= 64 lookups that
 * every rank runs with the same list; the answers are zg_lookup_subjects' on a replica. Shard r holds the forward rows
 * of the objects it owns, but their subjects can be owned by any shard: each level, every rank expands its own
 * frontier, routes the subjects it finds to their owners (one all-to-all), and the owner admits each object once per
 * lookup. Candidates are verified by the sharded check protocol, a second time with zg_shard_pass_nowild_dev when
 * the wildcard is granted, and the answers are sent to the rank that asked the lookup. A round ends a LookupResources
 * round begun on the same engine, and the other way round. Same conventions as the zg_shard_lookup_*_dev calls.
 *   zg_shard_pass_nowild_dev         zg_shard_pass_dev with every wildcard relationship invisible
 *   zg_shard_subjects_begin_dev      starts a round: res_types, reqs (res, perm of that type, stype, srel), options
 *                                    (ZG_WILDCARDS_*) and home (rank that asked) are HOST arrays of k; the
 *                                    owner of each resource puts it in d_front (device, walk_cap entries, *n_front)
 *   zg_shard_subjects_expand_dev     expands the n_in entries of this rank's frontier d_front over its forward rows;
 *                                    the subjects found go to d_routed (walk_cap entries) bucketed by owner (id % n_dest),
 *                                    counts[d] (HOST, n_dest); *overflow = 1 when an outbox, a frontier or the
 *                                    candidates did not fit in this round so far (redo it in halves; a single lookup
 *                                    verifies every object of the subject type instead), and nothing is routed
 *   zg_shard_subjects_admit_dev      the n_in entries that arrived from every rank -> the fresh ones in d_next
 *                                    (walk_cap entries), *n_next; fresh objects of the subject type become candidates
 *   zg_shard_subjects_candidates_dev this rank's check items: the probe of each owned resource (subject
 *                                    ZG_NO_OBJECT - 1), then the walk's candidates, or with exhaustive every owned id
 *                                    of the subject type; with d_items NULL, *n = the capacity needed; ZG_E2BIG when
 *                                    cap is smaller
 *   zg_shard_subjects_verdicts_dev   d_codes (one per item) -> *granted bit i: lookup i's probe checks HAS without a
 *                                    subject relation; *failed bit i: an item of lookup i is undecidable (ZG_EDEPTH)
 *   zg_shard_subjects_nowild_dev     with every rank's masks OR-ed: the HAS candidates of granted lookups -> d_items
 *                                    (cap >= the candidates), *n_nw, for the no-wildcards verification
 *   zg_shard_subjects_route_dev      d_codes of that verification (one per item) -> answer keys (excluded << 38 |
 *                                    lookup << 32 | id) in d_routed (the candidates' count), bucketed by home rank;
 *                                    counts[d] (HOST, n_dest)
 *   zg_shard_subjects_finish_dev     the keys that arrived home -> d_ids: the listed ids of lookup 0, 1, ... then the
 *                                    excluded ids of lookup 0, 1, ..., ascending each; listed[i] / excluded[i] (HOST,
 *                                    k) = their counts. The wildcard entry of lookup i is present when it is granted,
 *                                    not failed, and asked for with ZG_WILDCARDS_INCLUDE. */
int zg_shard_pass_nowild_dev(zg_engine *e, const zg_check *d_queries, uint64_t n, int level, uint64_t *n_sub);
int zg_shard_subjects_begin_dev(zg_engine *e, const uint16_t *res_types, const zg_check *reqs, const uint32_t *options,
                                const uint8_t *home, uint32_t k, uint64_t walk_cap, uint64_t *d_front, uint64_t *n_front);
int zg_shard_subjects_expand_dev(zg_engine *e, const uint64_t *d_front, uint64_t n_in, uint32_t n_dest, uint64_t *d_routed,
                                 uint64_t *counts, int *overflow);
int zg_shard_subjects_admit_dev(zg_engine *e, const uint64_t *d_in, uint64_t n_in, uint64_t *d_next, uint64_t *n_next);
int zg_shard_subjects_candidates_dev(zg_engine *e, int exhaustive, zg_check *d_items, uint64_t cap, uint64_t *n);
int zg_shard_subjects_verdicts_dev(zg_engine *e, const uint8_t *d_codes, uint64_t n, uint64_t *granted, uint64_t *failed);
int zg_shard_subjects_nowild_dev(zg_engine *e, const uint8_t *d_codes, uint64_t n, uint64_t granted, uint64_t failed,
                                 zg_check *d_items, uint64_t cap, uint64_t *n_nw);
int zg_shard_subjects_route_dev(zg_engine *e, const uint8_t *d_codes, uint64_t n, uint32_t n_dest, uint64_t *d_routed,
                                uint64_t *counts);
int zg_shard_subjects_finish_dev(zg_engine *e, const uint64_t *d_keys, uint64_t n, uint32_t *d_ids, uint64_t *listed,
                                 uint64_t *excluded);

/* Watch feed (v1.WatchServiceClient.Watch, pkg/authz/watch.go:27-48): the relationship changes made
 * visible by revisions > since_revision, oldest first, as '\n'-separated lines
 *   "<revision> <TOUCH|CREATE|DELETE> <type:id#rel@stype:sid[#srel]>[ <expires_at>]"
 * restricted to resources of res_type (NULL/"" = all; WatchRequest.OptionalObjectTypes). Only
 * zg_write_relationships / zg_delete_relationships feed it (interned bulk loads do not); a DELETE
 * of a relationship that did not exist is not a change. *through_revision = the engine's current
 * revision: pass it as the next since_revision. ZG_EPRECOND when since_revision is older than the
 * retained feed (2^20 changes), ZG_E2BIG with *need = bytes required incl. NUL. */
int zg_watch_read(zg_engine *e, uint64_t since_revision, const char *res_type, char *buf, size_t cap,
                  size_t *need, uint64_t *n_out, uint64_t *through_revision);

/* ---- list-response filter (SURVEY.md 8(f) rank 1; host code, no GPU) -------
 * Replaces the unmarshal / re-marshal round trip of pkg/authz/postfilter.go:17-55
 * (filterListResponse) and the name extraction of postfilter.go:67-119: one structural pass
 * over the body, then a splice of the kept items' bytes. */
typedef struct zg_list_item {
  uint64_t begin, end;  /* byte range of the item's JSON value inside the body           */
  uint64_t name_off;    /* metadata.name: offset of the string CONTENTS (still escaped)  */
  uint64_t ns_off;      /* metadata.namespace, same                                      */
  uint32_t name_len;    /* 0 = absent or not a string                                    */
  uint32_t ns_len;
  uint32_t flags;       /* ZG_ITEM_*                                                     */
  uint32_t reserved;
} zg_list_item;
#define ZG_ITEM_IS_OBJECT 1u    /* the item is a JSON object (others are never checked)  */
#define ZG_ITEM_HAS_METADATA 2u /* ... with an object-valued "metadata"                  */
#define ZG_ITEM_HAS_OBJECT 4u   /* table rows: the row has an "object" key (any value)   */
#define ZG_ITEM_RAW_NAMES 8u    /* name / namespace ranges are plain bytes (protobuf), not escaped JSON */
#define ZG_LIST_ITEMS 0u        /* scan "items"; metadata at item level                  */
#define ZG_LIST_TABLE_ROWS 1u   /* scan "rows"; metadata under rows[i].object (metav1.Table,
                                   pkg/authz/responsefilterer.go:349-374)                */
#define ZG_LIST_PROTOBUF 2u     /* a protobuf-encoded <Kind>List (Content-Type application/vnd.kubernetes.protobuf,
                                   pkg/authz/responsefilterer.go:256-266,:301-313): magic "k8s\0", runtime.Unknown,
                                   raw = { ListMeta metadata = 1; repeated <Kind> items = 2 }. Items: begin/end =
                                   the whole `items` entry (tag, length, message), names = plain bytes;
                                   *items_begin = offset of raw's length varint, *items_end = end of raw. Only
                                   the pre-filter has a protobuf path in the reference (the post-filter
                                   json.Unmarshals the body, postfilter.go:19). */
#define ZG_LIST_PROTOBUF_OBJECT 3u /* zg_list_scan only: ONE protobuf-encoded object (a get: responsefilterer.go:320-341,
                                     filterObject :403-415): a single item = the raw payload, with its names; the
                                     caller passes the body through or answers "unauthorized" */
#define ZG_LIST_EMPTY_AS_NULL 1u /* zg_list_filter flag: nothing kept -> null, not []    */
/* Scans a kube List (or Table) body. Returns the number of elements of the top-level "items" ("rows") array
 * (0 if there is no such array: the reference then passes the body through), ZG_EINVAL on
 * malformed JSON, ZG_E2BIG if out != NULL and cap is too small. [*items_begin, *items_end) is
 * the byte range of the array, brackets included. */
int64_t zg_list_scan(const char *body, size_t len, uint32_t mode, zg_list_item *out, uint64_t cap,
                     uint64_t *items_begin, uint64_t *items_end);
/* Writes the body with only the items whose keep[i] != 0; every other byte is preserved.
 * A protobuf body (recognised by its magic) loses the dropped `items` entries and gets the length of `raw` rewritten;
 * pass the items_begin / items_end its scan returned. With nothing kept the JSON array becomes `[]` (the pre-filter's filterList / filterTable,
 * responsefilterer.go:356,377) or, with ZG_LIST_EMPTY_AS_NULL, `null` (the post-filter's re-marshal of
 * a nil slice, postfilter.go:138). Returns 0, or ZG_E2BIG with *out_len = bytes required. */
int zg_list_filter(const char *body, size_t len, const zg_list_item *items, uint64_t n,
                   const uint8_t *keep, uint64_t items_begin, uint64_t items_end, uint32_t flags,
                   char *out, size_t cap, size_t *out_len);

/* The standard post-filter template, `T:{{namespacedName}}#perm@S:subject` (or `{{name}}`), for a
 * whole scanned list at once: no per-item strings cross the boundary. */
typedef struct zg_list_template {
  const char *res_type, *permission;           /* literal fields of the template                */
  const char *subj_type, *subj_id, *subj_rel;  /* the (already resolved) subject                */
  const char *req_name, *req_namespace;        /* request fallbacks (pkg/rules/rules.go:321-326);
                                                  NULL = ""                                     */
  uint32_t id_kind;                            /* ZG_ID_NAME | ZG_ID_NAMESPACED_NAME            */
  uint32_t flags;                              /* ZG_TPL_CLEAR_NAMESPACE                        */
} zg_list_template;
#define ZG_ID_NAME 0u            /* resource id = {{name}}                                      */
#define ZG_ID_NAMESPACED_NAME 1u /* resource id = "namespace/name", or "name" without namespace  */
#define ZG_TPL_CLEAR_NAMESPACE 1u /* the request is on `namespaces` (rules.go:331-333)           */
/* Builds one interned check per scanned item straight from the body bytes (JSON escapes decoded).
 * checked[i] = 0 for items the reference never checks (not an object: postfilter.go:68-71) or whose
 * resource id comes out empty (the template does not resolve: :91-95); their out[i] is a placeholder
 * and the caller keeps them. No GPU work: feed out[] to zg_check_bulk. */
int zg_list_resolve(zg_engine *e, const char *body, size_t len, const zg_list_item *items, uint64_t n,
                    const zg_list_template *tpl, zg_check *out, uint8_t *checked);
/* Scan + resolve + ONE bulk check + splice, for a post-filter made of `n_tpl` such templates (an item
 * is kept when every template answers HAS_PERMISSION, postfilter.go:149-170). Returns 0 with the
 * filtered body in out (or the body itself, copied, when the reference would pass it through),
 * ZG_E2BIG with *out_len = bytes required, ZG_EINVAL on a malformed body. */
int zg_list_postfilter(zg_engine *e, const char *body, size_t len, const zg_list_template *tpl,
                       uint32_t n_tpl, char *out, size_t cap, size_t *out_len);

/* The pre-filter side of the same scan (pkg/authz/lookups.go:44-132 + responsefilterer.go:349-400):
 * keep[i] = 1 when the item's (namespace, name) is what an allowed resource id maps to under the usual
 * id <-> name rule ("namespace/name" -> (namespace, name); "name" -> (request namespace or "", name)).
 * `allowed` = object ids of res_type, ascending, as zg_lookup_resources returns them; self_name
 * (NULL = none) is one more allowed id given by name. mode = ZG_LIST_ITEMS | ZG_LIST_TABLE_ROWS. An
 * element that is not an object, or a table row without "object", is ZG_EINVAL (the reference fails to
 * decode such a body). No GPU work. */
int zg_list_keep_allowed(zg_engine *e, const char *body, size_t len, const zg_list_item *items, uint64_t n,
                         uint32_t mode, const char *res_type, const char *req_namespace,
                         const uint32_t *allowed, uint64_t n_allowed, const char *self_name, uint8_t *keep);
/* LookupResources (tpl's literal fields; id_kind / req_name are not used) + scan + keep + splice: the
 * whole pre-filtered List or Table response in one call. Nothing kept gives [] here. */
int zg_list_prefilter(zg_engine *e, const char *body, size_t len, uint32_t mode, const zg_list_template *tpl,
                      char *out, size_t cap, size_t *out_len);

/* ---- measurement --------------------------------------------------------- */
/* Build time and tuning macros of this library (goes into every bench line). */
const char *zg_build_info(void);
int zg_stats_get(zg_engine *e, zg_stats *out);
/* Runs the batch through the instrumented kernel variant and returns the
 * ALGORITHMIC bytes it needed (DESIGN.md "Algorithmic bytes"); not for timing. */
int zg_count_alg_bytes(zg_engine *e, const zg_check *items, uint64_t n, uint64_t *bytes);

/* Cumulative clock64() cycles the check kernel's warps spent per phase since the engine was created:
 * admission, root visit, two-level meet, one-level meet, pop loop (the visits exclude the meets inside them).
 * Only a library built with -DZG_PHASE_CLOCKS=1 counts them; any other build returns ZG_EINVAL. */
int zg_phase_clocks(zg_engine *e, uint64_t cycles[5]);

#ifdef __cplusplus
}
#endif
#endif
