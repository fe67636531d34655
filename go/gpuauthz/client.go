// Package gpuauthz is the reference-side binding of libzgpu: an implementation of
// v1.PermissionsServiceClient (authzed-go v1.6.0) that answers CheckPermission,
// CheckBulkPermissions and LookupResources on an H100 through the C ABI in
// include/zgpu.h, and delegates everything else to the embedded SpiceDB it wraps.
//
// Injection point in the reference: pkg/proxy/options.go:371-377 only assigns
// Options.PermissionsClient when it is nil, so
//
//	opts.PermissionsClient = gpuauthz.New(embeddedClient, schemaText)
//
// before opts.Complete() is all the proxy needs (pkg/proxy/server.go:136-139,153 pass
// the same client to the workflow activities and to pkg/authz).
//
// STATUS: written against the v1 API from the call sites in the reference
// (pkg/authz/check.go:23-69, lookups.go:49-88, watch.go:50-67, postfilter.go:97-172,
// distributedtx/activity.go:54-171). It has NOT been compiled: there is no Go toolchain
// in the build image or on the GPU box. The Python mirror
// (spicedb-kubeapi-proxy_b200/client.py) drives the identical C ABI in the tests.
package gpuauthz

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../spicedb-kubeapi-proxy_b200 -lzgpu -Wl,-rpath,${SRCDIR}/../../spicedb-kubeapi-proxy_b200
#include <stdlib.h>
#include <string.h>
#include "zgpu.h"

static zg_rel_str *rel_array(size_t n) { return (zg_rel_str *)calloc(n ? n : 1, sizeof(zg_rel_str)); }
static zg_update_str *upd_array(size_t n) { return (zg_update_str *)calloc(n ? n : 1, sizeof(zg_update_str)); }
static zg_precondition_str *pre_array(size_t n) { return (zg_precondition_str *)calloc(n ? n : 1, sizeof(zg_precondition_str)); }
*/
import "C"

import (
	"context"
	"encoding/base64"
	"fmt"
	"io"
	"runtime"
	"strconv"
	"strings"
	"sync"
	"sync/atomic"
	"time"
	"unsafe"

	v1 "github.com/authzed/authzed-go/proto/authzed/api/v1"
	"google.golang.org/grpc"
	"google.golang.org/grpc/codes"
	"google.golang.org/grpc/metadata"
	"google.golang.org/grpc/status"
)

// Client implements v1.PermissionsServiceClient.
type Client struct {
	v1.PermissionsServiceClient // the embedded SpiceDB: source of truth for everything not overridden

	engine *C.zg_engine
	mu     sync.Mutex // serialises the write mirror; checks are thread-safe in the library
	// broken is set when the mirror diverged from SpiceDB and could not be rebuilt: every check path
	// then fails (pkg/authz/authz.go:93-97 turns an error into a denial) instead of answering from a
	// store that may still hold revoked grants.
	broken atomic.Bool
	// sharded: the engine is a sharded handle (Shards), which answers checks and writes but refuses LookupResources
	// unless HandleLookups is set, and LookupSubjects unless HandleSubjects is set; what it refuses goes to the
	// embedded SpiceDB
	sharded, handleLookups, handleSubjects bool
}

// AllDevices: every visible GPU from `device` on (zg_config.n_devices).
const AllDevices = uint32(C.ZG_ALL_DEVICES)

// Option adjusts the engine's configuration before it is created.
type Option func(*C.zg_config)

// Shards makes the one engine hold the n shards of an object-hash sharded store (zg_config.n_shards): shard k keeps
// the relationships whose resource id % n == k and lives on device `device + k % nDevices` (with nDevices = 1, the n
// shards share one GPU). For stores larger than one GPU. Checks and writes are answered by the engine;
// LookupResources and LookupSubjects are delegated to the embedded SpiceDB unless HandleLookups / HandleSubjects
// is set.
func Shards(n uint32) Option {
	return func(cfg *C.zg_config) { cfg.n_shards = C.uint32_t(n) }
}

// HandleLookups, with Shards, makes the sharded engine answer LookupResources and PrefilterListResponse itself
// (ZG_FLAG_HANDLE_LOOKUPS): the reverse walk runs on every shard and the answers equal a replica's, so a store larger
// than one GPU serves pre-filtered lists without a second engine. LookupSubjects stays delegated unless
// HandleSubjects is set too.
func HandleLookups() Option {
	return func(cfg *C.zg_config) { cfg.flags |= C.ZG_FLAG_HANDLE_LOOKUPS }
}

// HandleSubjects, with Shards, makes the sharded engine answer LookupSubjects itself (ZG_FLAG_HANDLE_SUBJECTS): the
// forward walk runs on every shard, each discovery sent to its owner, and the answers equal a replica's. Independent
// of HandleLookups.
func HandleSubjects() Option {
	return func(cfg *C.zg_config) { cfg.flags |= C.ZG_FLAG_HANDLE_SUBJECTS }
}

var errBroken = status.Error(codes.Unavailable, "gpu mirror is out of sync with SpiceDB and could not be rebuilt")

// New creates the GPU engine, loads the schema and mirrors the relationships that are
// already in SpiceDB (bootstrap file: pkg/spicedb/spicedb.go:19-24).
//
// nDevices > 1 (or AllDevices) makes the one engine own that many GPUs of the box, each holding a replica of the
// snapshot and answering its slice of every bulk call: the proxy keeps a single client (pkg/proxy/options.go:81-82),
// so this is how it uses more than one GPU.
func New(ctx context.Context, inner v1.PermissionsServiceClient, schema string, device int, nDevices uint32, opts ...Option) (*Client, error) {
	cfg := C.zg_config{device: C.int32_t(device), n_devices: C.uint32_t(nDevices)}
	for _, o := range opts {
		o(&cfg)
	}
	var eng *C.zg_engine
	if err := call(func() C.int { return C.zg_engine_create(&cfg, &eng) }); err != nil {
		return nil, err // fail closed: no CPU fallback inside the library
	}
	c := &Client{PermissionsServiceClient: inner, engine: eng, sharded: cfg.n_shards > 1,
		handleLookups: cfg.flags&C.ZG_FLAG_HANDLE_LOOKUPS != 0, handleSubjects: cfg.flags&C.ZG_FLAG_HANDLE_SUBJECTS != 0}
	cs := C.CString(schema)
	defer C.free(unsafe.Pointer(cs))
	if err := call(func() C.int { return C.zg_load_schema(eng, cs, C.size_t(len(schema))) }); err != nil {
		c.Close()
		return nil, err
	}
	if err := c.resync(ctx); err != nil {
		c.Close()
		return nil, err
	}
	return c, nil
}

func (c *Client) Close() {
	if c.engine != nil {
		C.zg_engine_destroy(c.engine)
		c.engine = nil
	}
}

// call runs one C entry point and, when it fails, fetches the library's message. zg_last_error is
// thread-local; a goroutine may migrate between OS threads from one cgo call to the next, so the pair
// (failing call, zg_last_error) runs with the goroutine pinned to its thread.
func call(f func() C.int) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	if rc := f(); rc != 0 {
		return lastError(rc)
	}
	return nil
}

// lastError must run on the OS thread of the failing call: only use it through call().
func lastError(rc C.int) error {
	code := codes.Internal
	switch rc {
	case C.ZG_EINVAL:
		code = codes.InvalidArgument
	case C.ZG_EEXIST:
		code = codes.AlreadyExists
	case C.ZG_EPRECOND, C.ZG_ENOSCHEMA, C.ZG_ENOSNAPSHOT:
		code = codes.FailedPrecondition
	case C.ZG_ENOMEM, C.ZG_EDEPTH:
		code = codes.ResourceExhausted
	}
	return status.Error(code, C.GoString(C.zg_last_error()))
}

// cstrs owns the C strings of one call.
type cstrs struct{ p []unsafe.Pointer }

func (s *cstrs) add(v string) *C.char {
	c := C.CString(v)
	s.p = append(s.p, unsafe.Pointer(c))
	return c
}
func (s *cstrs) free() {
	for _, p := range s.p {
		C.free(p)
	}
}

func (s *cstrs) fillRel(dst *C.zg_rel_str, res *v1.ObjectReference, relation string, subj *v1.SubjectReference) {
	dst.res_type = s.add(res.GetObjectType())
	dst.res_id = s.add(res.GetObjectId())
	dst.relation = s.add(relation)
	dst.subj_type = s.add(subj.GetObject().GetObjectType())
	dst.subj_id = s.add(subj.GetObject().GetObjectId())
	dst.subj_rel = s.add(subj.GetOptionalRelation())
}

// fillFilterEx: fillFilter and optional_resource_id_prefix ("" = unset).
func (s *cstrs) fillFilterEx(dst *C.zg_filter_ex, f *v1.RelationshipFilter) {
	s.fillFilter(&dst.f, f)
	dst.res_id_prefix = s.add(f.GetOptionalResourceIdPrefix())
}

func (s *cstrs) fillFilter(dst *C.zg_filter_str, f *v1.RelationshipFilter) {
	dst.res_type = s.add(f.GetResourceType())
	dst.res_id = s.add(f.GetOptionalResourceId())
	dst.relation = s.add(f.GetOptionalRelation())
	if sf := f.GetOptionalSubjectFilter(); sf != nil {
		dst.subj_type = s.add(sf.GetSubjectType())
		dst.subj_id = s.add(sf.GetOptionalSubjectId())
		if r := sf.GetOptionalRelation(); r != nil {
			rel := r.GetRelation()
			if rel == "" {
				rel = "..."
			}
			dst.subj_rel = s.add(rel)
		}
	}
}

// CheckBulkPermissions: pkg/authz/check.go:41-69 and postfilter.go:127-178 rely on
// Pairs[i] answering Items[i], and only on == PERMISSIONSHIP_HAS_PERMISSION.
func (c *Client) CheckBulkPermissions(ctx context.Context, req *v1.CheckBulkPermissionsRequest, _ ...grpc.CallOption) (*v1.CheckBulkPermissionsResponse, error) {
	n := len(req.GetItems())
	resp := &v1.CheckBulkPermissionsResponse{Pairs: make([]*v1.CheckBulkPermissionsPair, n)}
	if n == 0 {
		return resp, nil
	}
	var s cstrs
	defer s.free()
	arr := C.rel_array(C.size_t(n))
	defer C.free(unsafe.Pointer(arr))
	items := unsafe.Slice(arr, n)
	for i, it := range req.GetItems() {
		s.fillRel(&items[i], it.GetResource(), it.GetPermission(), it.GetSubject())
	}
	out := (*C.uint8_t)(C.malloc(C.size_t(n)))
	defer C.free(unsafe.Pointer(out))
	if c.broken.Load() {
		return nil, errBroken
	}
	if err := call(func() C.int { return C.zg_check_bulk_str(c.engine, arr, C.uint64_t(n), out) }); err != nil {
		return nil, err // fail closed: pkg/authz/authz.go:93-97 turns any error into a denial
	}
	codesOut := unsafe.Slice((*byte)(unsafe.Pointer(out)), n)
	for i, it := range req.GetItems() {
		pair := &v1.CheckBulkPermissionsPair{Request: it}
		if codesOut[i] == C.ZG_ITEM_ERROR {
			pair.Response = &v1.CheckBulkPermissionsPair_Error{Error: status.New(codes.FailedPrecondition,
				"check failed: unknown permission or type, or maximum depth exceeded").Proto()}
		} else {
			pair.Response = &v1.CheckBulkPermissionsPair_Item{Item: &v1.CheckBulkPermissionsResponseItem{
				Permissionship: v1.CheckPermissionResponse_Permissionship(codesOut[i])}}
		}
		resp.Pairs[i] = pair
	}
	return resp, nil
}

// CheckPermission: pkg/authz/watch.go:50-67 (one call per relationship update).
func (c *Client) CheckPermission(ctx context.Context, req *v1.CheckPermissionRequest, opts ...grpc.CallOption) (*v1.CheckPermissionResponse, error) {
	bulk, err := c.CheckBulkPermissions(ctx, &v1.CheckBulkPermissionsRequest{
		Consistency: req.GetConsistency(),
		Items: []*v1.CheckBulkPermissionsRequestItem{{
			Resource: req.GetResource(), Permission: req.GetPermission(), Subject: req.GetSubject()}},
	}, opts...)
	if err != nil {
		return nil, err
	}
	if e := bulk.Pairs[0].GetError(); e != nil {
		return nil, status.ErrorProto(e)
	}
	return &v1.CheckPermissionResponse{Permissionship: bulk.Pairs[0].GetItem().GetPermissionship()}, nil
}

// LookupResources: pkg/authz/lookups.go:65-88 reads the stream until io.EOF and keeps
// LOOKUP_PERMISSIONSHIP_HAS_PERMISSION entries; order is irrelevant (a set).
func (c *Client) LookupResources(ctx context.Context, req *v1.LookupResourcesRequest, opts ...grpc.CallOption) (v1.PermissionsService_LookupResourcesClient, error) {
	if c.sharded && !c.handleLookups {
		return c.PermissionsServiceClient.LookupResources(ctx, req, opts...)
	}
	if c.broken.Load() {
		return nil, errBroken
	}
	if req.GetOptionalLimit() != 0 || req.GetOptionalCursor() != nil {
		return c.lookupResourcesPaged(ctx, req)
	}
	var s cstrs
	defer s.free()
	subj := req.GetSubject()
	capacity := C.size_t(1 << 16)
	for {
		buf := (*C.char)(C.malloc(capacity))
		var need C.size_t
		var n C.uint64_t
		var rc C.int
		err := call(func() C.int {
			rc = C.zg_lookup_resources_str(c.engine, s.add(req.GetResourceObjectType()), s.add(req.GetPermission()),
				s.add(subj.GetObject().GetObjectType()), s.add(subj.GetObject().GetObjectId()),
				s.add(subj.GetOptionalRelation()), buf, capacity, &need, &n)
			if rc == C.ZG_E2BIG {
				return 0
			}
			return rc
		})
		if rc == C.ZG_E2BIG {
			C.free(unsafe.Pointer(buf))
			capacity = need + 16
			continue
		}
		if err != nil {
			C.free(unsafe.Pointer(buf))
			return nil, err
		}
		ids := strings.Split(strings.TrimSuffix(C.GoString(buf), "\n"), "\n")
		C.free(unsafe.Pointer(buf))
		if n == 0 {
			ids = nil
		}
		return &sliceStream{ctx: ctx, ids: ids}, nil
	}
}

// lookupResourcesPaged answers a LookupResources with OptionalLimit or OptionalCursor through
// zg_lookup_resources_page_str: with a limit, one page of at most OptionalLimit resources after the cursor; with only
// a cursor, every resource after it. Resources come in ascending interned id order (SpiceDB promises no order), each
// with the AfterResultCursor that resumes after it. The cursor token is the base64 of the engine's 32 opaque bytes.
func (c *Client) lookupResourcesPaged(ctx context.Context, req *v1.LookupResourcesRequest) (v1.PermissionsService_LookupResourcesClient, error) {
	var s cstrs
	defer s.free()
	subj := req.GetSubject()
	var cur *C.zg_read_cursor
	if tok := req.GetOptionalCursor().GetToken(); tok != "" {
		raw, err := base64.StdEncoding.DecodeString(tok)
		if err != nil || len(raw) != C.ZG_READ_CURSOR_BYTES {
			return nil, status.Errorf(codes.InvalidArgument, "lookup cursor: not a cursor of this engine")
		}
		cur = (*C.zg_read_cursor)(C.CBytes(raw))
		defer C.free(unsafe.Pointer(cur))
	}
	limit := uint64(req.GetOptionalLimit())
	page := limit
	if page == 0 || page > 1<<16 { // no limit: pages of 1 000; a larger limit is cut into pages of 1 << 16
		page = 1000
		if limit != 0 {
			page = 1 << 16
		}
	}
	st := &sliceStream{ctx: ctx}
	for capBytes := uint64(1 << 16); ; {
		buf := C.malloc(C.size_t(capBytes))
		curs := make([]C.zg_read_cursor, page+1)
		var need C.size_t
		var n C.uint64_t
		var next C.zg_read_cursor
		var more C.int32_t
		big := false
		err := call(func() C.int {
			rc := C.zg_lookup_resources_page_str(c.engine, s.add(req.GetResourceObjectType()), s.add(req.GetPermission()),
				s.add(subj.GetObject().GetObjectType()), s.add(subj.GetObject().GetObjectId()), s.add(subj.GetOptionalRelation()),
				C.uint64_t(page), cur, (*C.char)(buf), C.size_t(capBytes), &need, &n, &curs[0], &next, &more)
			big = rc == C.ZG_E2BIG
			if big {
				return 0
			}
			return rc
		})
		if err != nil || big {
			C.free(buf)
			if err != nil {
				return nil, err
			}
			capBytes = uint64(need) + 16
			continue
		}
		text := C.GoString((*C.char)(buf))
		C.free(buf)
		if text != "" {
			for i, id := range strings.Split(strings.TrimSuffix(text, "\n"), "\n") {
				st.ids = append(st.ids, id)
				st.cursors = append(st.cursors, base64.StdEncoding.EncodeToString(C.GoBytes(unsafe.Pointer(&curs[i]), C.ZG_READ_CURSOR_BYTES)))
			}
		}
		done := more == 0
		if limit != 0 {
			limit -= uint64(n)
			done = done || limit == 0
			if limit < page {
				page = limit
			}
		}
		if done {
			return st, nil
		}
		if cur == nil {
			cur = (*C.zg_read_cursor)(C.malloc(C.ZG_READ_CURSOR_BYTES))
			defer C.free(unsafe.Pointer(cur))
		}
		*cur = next
	}
}

type sliceStream struct {
	ctx     context.Context
	ids     []string
	cursors []string // AfterResultCursor tokens of a paged lookup (nil: unpaged)
	pos     int
}

func (s *sliceStream) Recv() (*v1.LookupResourcesResponse, error) {
	if err := s.ctx.Err(); err != nil {
		return nil, status.FromContextError(err).Err() // codes.Canceled is special-cased at responsefilterer.go:170
	}
	if s.pos >= len(s.ids) {
		return nil, io.EOF
	}
	id := s.ids[s.pos]
	r := &v1.LookupResourcesResponse{ResourceObjectId: id,
		Permissionship: v1.LookupPermissionship_LOOKUP_PERMISSIONSHIP_HAS_PERMISSION}
	if s.cursors != nil {
		r.AfterResultCursor = &v1.Cursor{Token: s.cursors[s.pos]}
	}
	s.pos++
	return r, nil
}
func (s *sliceStream) Header() (metadata.MD, error) { return nil, nil }
func (s *sliceStream) Trailer() metadata.MD         { return nil }
func (s *sliceStream) CloseSend() error             { return nil }
func (s *sliceStream) Context() context.Context     { return s.ctx }
func (s *sliceStream) SendMsg(any) error            { return nil }
func (s *sliceStream) RecvMsg(any) error            { return io.EOF }

// LookupSubjects: "which subjects of a type have the permission on this resource" (who-can / audit). No proxy
// call site issues it (it is in the client mock of pkg/authz/postfilter_test.go:71). A request with caveat
// context, a concrete limit or a cursor goes to the wrapped SpiceDB: the library answers whole, uncaveated
// lookups only, and a sharded engine only with HandleSubjects. The concrete subjects come first, then -- when a
// wildcard grants the permission and the request includes wildcards -- "*" with its excluded subjects. Like the
// rest of this file: never compiled.
func (c *Client) LookupSubjects(ctx context.Context, req *v1.LookupSubjectsRequest, opts ...grpc.CallOption) (v1.PermissionsService_LookupSubjectsClient, error) {
	if (c.sharded && !c.handleSubjects) || req.GetContext() != nil || req.GetOptionalConcreteLimit() != 0 || req.GetOptionalCursor() != nil {
		return c.PermissionsServiceClient.LookupSubjects(ctx, req, opts...)
	}
	if c.broken.Load() {
		return nil, errBroken
	}
	var s cstrs
	defer s.free()
	option := C.uint32_t(C.ZG_WILDCARDS_INCLUDE)
	if req.GetWildcardOption() == v1.LookupSubjectsRequest_WILDCARD_OPTION_EXCLUDE_WILDCARDS {
		option = C.ZG_WILDCARDS_EXCLUDE
	}
	capacity := C.size_t(1 << 16)
	for {
		buf := (*C.char)(C.malloc(capacity))
		var need C.size_t
		var n C.uint64_t
		var rc C.int
		err := call(func() C.int {
			rc = C.zg_lookup_subjects_str(c.engine, s.add(req.GetResource().GetObjectType()),
				s.add(req.GetResource().GetObjectId()), s.add(req.GetPermission()), s.add(req.GetSubjectObjectType()),
				s.add(req.GetOptionalSubjectRelation()), option, buf, capacity, &need, &n)
			if rc == C.ZG_E2BIG {
				return 0
			}
			return rc
		})
		if rc == C.ZG_E2BIG {
			C.free(unsafe.Pointer(buf))
			capacity = need + 16
			continue
		}
		if err != nil {
			C.free(unsafe.Pointer(buf))
			return nil, err
		}
		lines := strings.Split(strings.TrimSuffix(C.GoString(buf), "\n"), "\n")
		C.free(unsafe.Pointer(buf))
		if n == 0 {
			lines = nil
		}
		var out []*v1.LookupSubjectsResponse
		has := v1.LookupPermissionship_LOOKUP_PERMISSIONSHIP_HAS_PERMISSION
		for i := 0; i < len(lines); i++ {
			if lines[i] != "*" {
				out = append(out, &v1.LookupSubjectsResponse{Subject: &v1.ResolvedSubject{SubjectObjectId: lines[i], Permissionship: has}})
				continue
			}
			wild := &v1.LookupSubjectsResponse{Subject: &v1.ResolvedSubject{SubjectObjectId: "*", Permissionship: has}}
			for _, x := range lines[i+1:] { // "!<id>": '!' is outside SpiceDB's object-id charset
				wild.ExcludedSubjects = append(wild.ExcludedSubjects, &v1.ResolvedSubject{SubjectObjectId: strings.TrimPrefix(x, "!"), Permissionship: has})
			}
			out = append(out, wild)
			break
		}
		return &subjectStream{ctx: ctx, items: out}, nil
	}
}

type subjectStream struct {
	ctx   context.Context
	items []*v1.LookupSubjectsResponse
	pos   int
}

func (s *subjectStream) Recv() (*v1.LookupSubjectsResponse, error) {
	if err := s.ctx.Err(); err != nil {
		return nil, status.FromContextError(err).Err()
	}
	if s.pos >= len(s.items) {
		return nil, io.EOF
	}
	s.pos++
	return s.items[s.pos-1], nil
}
func (s *subjectStream) Header() (metadata.MD, error) { return nil, nil }
func (s *subjectStream) Trailer() metadata.MD         { return nil }
func (s *subjectStream) CloseSend() error             { return nil }
func (s *subjectStream) Context() context.Context     { return s.ctx }
func (s *subjectStream) SendMsg(any) error            { return nil }
func (s *subjectStream) RecvMsg(any) error            { return io.EOF }

// ExpandPermissionTree: the permission's subject tree at the resource, built on the GPU from zg_expand_permission_tree_str
// (one line per node in pre-order: "<depth> <U|I|X|L> <type>:<id>#<relation>[ <subject>]*"). A sharded engine delegates
// to the embedded SpiceDB.
func (c *Client) ExpandPermissionTree(ctx context.Context, req *v1.ExpandPermissionTreeRequest, opts ...grpc.CallOption) (*v1.ExpandPermissionTreeResponse, error) {
	if c.sharded {
		return c.PermissionsServiceClient.ExpandPermissionTree(ctx, req, opts...)
	}
	if c.broken.Load() {
		return nil, errBroken
	}
	var s cstrs
	defer s.free()
	capacity := C.size_t(1 << 16)
	for {
		buf := (*C.char)(C.malloc(capacity))
		var need C.size_t
		var n C.uint64_t
		var rc C.int
		err := call(func() C.int {
			rc = C.zg_expand_permission_tree_str(c.engine, s.add(req.GetResource().GetObjectType()),
				s.add(req.GetResource().GetObjectId()), s.add(req.GetPermission()), buf, capacity, &need, &n)
			if rc == C.ZG_E2BIG {
				return 0
			}
			return rc
		})
		if rc == C.ZG_E2BIG {
			C.free(unsafe.Pointer(buf))
			capacity = need + 16
			continue
		}
		if err != nil {
			C.free(unsafe.Pointer(buf))
			return nil, err
		}
		lines := strings.Split(strings.TrimSuffix(C.GoString(buf), "\n"), "\n")
		C.free(unsafe.Pointer(buf))
		ops := map[string]v1.AlgebraicSubjectSet_Operation{"U": v1.AlgebraicSubjectSet_OPERATION_UNION,
			"I": v1.AlgebraicSubjectSet_OPERATION_INTERSECTION, "X": v1.AlgebraicSubjectSet_OPERATION_EXCLUSION}
		ref := func(s string) (*v1.ObjectReference, string) { // "type:id[#rel]"
			t, rest, _ := strings.Cut(s, ":")
			id, rel, _ := strings.Cut(rest, "#")
			return &v1.ObjectReference{ObjectType: t, ObjectId: id}, rel
		}
		var root *v1.PermissionRelationshipTree
		var stack []*v1.PermissionRelationshipTree // the open ancestors of the next line, by depth
		for _, line := range lines {
			f := strings.Split(line, " ")
			depth, _ := strconv.Atoi(f[0])
			at := strings.LastIndex(f[2], "#")
			obj, _ := ref(f[2][:at])
			node := &v1.PermissionRelationshipTree{ExpandedObject: obj, ExpandedRelation: f[2][at+1:]}
			if f[1] == "L" {
				leaf := &v1.DirectSubjectSet{}
				for _, x := range f[3:] {
					o, rel := ref(x)
					leaf.Subjects = append(leaf.Subjects, &v1.SubjectReference{Object: o, OptionalRelation: rel})
				}
				node.TreeType = &v1.PermissionRelationshipTree_Leaf{Leaf: leaf}
			} else {
				node.TreeType = &v1.PermissionRelationshipTree_Intermediate{Intermediate: &v1.AlgebraicSubjectSet{Operation: ops[f[1]]}}
			}
			stack = stack[:depth]
			if depth == 0 {
				root = node
			} else {
				parent := stack[depth-1].GetIntermediate()
				parent.Children = append(parent.Children, node)
			}
			stack = append(stack, node)
		}
		return &v1.ExpandPermissionTreeResponse{TreeRoot: root}, nil
	}
}

// WriteRelationships: SpiceDB stays the source of truth (preconditions, idempotency keys
// with expiry: pkg/authz/distributedtx/activity.go:54-102); a successful write is mirrored
// into the GPU store before returning so FullyConsistent checks observe it.
func (c *Client) WriteRelationships(ctx context.Context, req *v1.WriteRelationshipsRequest, opts ...grpc.CallOption) (*v1.WriteRelationshipsResponse, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	resp, err := c.PermissionsServiceClient.WriteRelationships(ctx, req, opts...)
	if err != nil {
		return nil, err
	}
	if err := c.mirror(req.GetUpdates()); err != nil {
		// the stores diverged (SpiceDB committed, the mirror rejected the batch -- DELETEs included):
		// rebuild the mirror from SpiceDB rather than serve stale answers
		if rerr := c.resync(ctx); rerr != nil {
			c.broken.Store(true)
			return nil, status.Errorf(codes.Internal, "gpu mirror failed (%v) and resync failed: %v", err, rerr)
		}
	}
	return resp, nil
}

func (c *Client) mirror(updates []*v1.RelationshipUpdate) error {
	n := len(updates)
	if n == 0 {
		return nil
	}
	var s cstrs
	defer s.free()
	arr := C.upd_array(C.size_t(n))
	defer C.free(unsafe.Pointer(arr))
	ups := unsafe.Slice(arr, n)
	for i, u := range updates {
		r := u.GetRelationship()
		s.fillRel(&ups[i].rel, r.GetResource(), r.GetRelation(), r.GetSubject())
		if ts := r.GetOptionalExpiresAt(); ts != nil {
			ups[i].expires_at = C.uint32_t(ts.GetSeconds())
		}
		switch u.GetOperation() {
		case v1.RelationshipUpdate_OPERATION_CREATE, v1.RelationshipUpdate_OPERATION_TOUCH:
			ups[i].op = C.ZG_OP_TOUCH // SpiceDB already enforced CREATE semantics
		case v1.RelationshipUpdate_OPERATION_DELETE:
			ups[i].op = C.ZG_OP_DELETE
		}
	}
	return call(func() C.int { return C.zg_write_relationships(c.engine, arr, C.uint64_t(n), nil, 0) })
}

// DeleteRelationships: delegate, then apply the same filter to the mirror.
func (c *Client) DeleteRelationships(ctx context.Context, req *v1.DeleteRelationshipsRequest, opts ...grpc.CallOption) (*v1.DeleteRelationshipsResponse, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	resp, err := c.PermissionsServiceClient.DeleteRelationships(ctx, req, opts...)
	if err != nil {
		return nil, err
	}
	var s cstrs
	defer s.free()
	var f C.zg_filter_ex
	s.fillFilterEx(&f, req.GetRelationshipFilter())
	if err := call(func() C.int { return C.zg_delete_relationships_limited_ex(c.engine, &f, nil, 0, 0, 0, nil, nil) }); err != nil {
		if rerr := c.resync(ctx); rerr != nil {
			c.broken.Store(true)
			return nil, status.Errorf(codes.Internal, "gpu mirror delete failed (%v) and resync failed: %v", err, rerr)
		}
	}
	return resp, nil
}

// CollectExpired removes from the mirror every relationship whose expiration is at or before `before`, which must
// not be later than the engine's clock, and returns how many it removed. Answers at any later time do not change and
// the watch feed records nothing; SpiceDB collects its own copy on its GC window. Nothing calls it automatically: run
// it periodically, e.g. every hour with time.Now().Add(-24 * time.Hour).
func (c *Client) CollectExpired(before time.Time) (uint64, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var n C.uint64_t
	if err := call(func() C.int { return C.zg_collect_expired(c.engine, C.int64_t(before.Unix()), &n) }); err != nil {
		return 0, err
	}
	return uint64(n), nil
}

// ImportBulkRelationships: the stream is buffered, forwarded to SpiceDB when the caller closes it, and on success
// imported into the mirror in one zg_import_relationships call (one group per class, packed ids: no C string per
// relationship). A mirror failure resyncs, as WriteRelationships does.
func (c *Client) ImportBulkRelationships(ctx context.Context, opts ...grpc.CallOption) (grpc.ClientStreamingClient[v1.ImportBulkRelationshipsRequest, v1.ImportBulkRelationshipsResponse], error) {
	inner, err := c.PermissionsServiceClient.ImportBulkRelationships(ctx, opts...)
	if err != nil {
		return nil, err
	}
	return &importStream{ClientStreamingClient: inner, c: c, ctx: ctx}, nil
}

type importStream struct {
	grpc.ClientStreamingClient[v1.ImportBulkRelationshipsRequest, v1.ImportBulkRelationshipsResponse]
	c    *Client
	ctx  context.Context
	rels []*v1.Relationship
}

func (s *importStream) Send(req *v1.ImportBulkRelationshipsRequest) error {
	s.rels = append(s.rels, req.GetRelationships()...)
	return s.ClientStreamingClient.Send(req)
}

func (s *importStream) CloseAndRecv() (*v1.ImportBulkRelationshipsResponse, error) {
	s.c.mu.Lock()
	defer s.c.mu.Unlock()
	resp, err := s.ClientStreamingClient.CloseAndRecv()
	if err != nil {
		return nil, err
	}
	if err := s.c.importMirror(s.rels); err != nil {
		if rerr := s.c.resync(s.ctx); rerr != nil {
			s.c.broken.Store(true)
			return nil, status.Errorf(codes.Internal, "gpu mirror failed (%v) and resync failed: %v", err, rerr)
		}
	}
	return resp, nil
}

// importMirror groups the relationships by class (first appearance of the class, then stream order) and imports them.
func (c *Client) importMirror(rels []*v1.Relationship) error {
	type group struct {
		rt, rel, st, srel string
		res, subj          []byte
		roff, soff         []C.uint32_t
		exp                []C.uint32_t
		expiring           bool
	}
	var order []*group
	byClass := map[[4]string]*group{}
	for _, r := range rels {
		k := [4]string{r.GetResource().GetObjectType(), r.GetRelation(), r.GetSubject().GetObject().GetObjectType(),
			r.GetSubject().GetOptionalRelation()}
		g := byClass[k]
		if g == nil {
			g = &group{rt: k[0], rel: k[1], st: k[2], srel: k[3], roff: []C.uint32_t{0}, soff: []C.uint32_t{0}}
			byClass[k] = g
			order = append(order, g)
		}
		g.res = append(g.res, r.GetResource().GetObjectId()...)
		g.subj = append(g.subj, r.GetSubject().GetObject().GetObjectId()...)
		g.roff = append(g.roff, C.uint32_t(len(g.res)))
		g.soff = append(g.soff, C.uint32_t(len(g.subj)))
		var e C.uint32_t
		if ts := r.GetOptionalExpiresAt(); ts != nil {
			e = C.uint32_t(ts.GetSeconds())
			g.expiring = true
		}
		g.exp = append(g.exp, e)
	}
	if len(order) == 0 {
		return nil
	}
	var s cstrs
	defer s.free()
	arr := (*C.zg_import_group)(C.calloc(C.size_t(len(order)), C.size_t(unsafe.Sizeof(C.zg_import_group{}))))
	defer C.free(unsafe.Pointer(arr))
	gs := unsafe.Slice(arr, len(order))
	for i, g := range order {
		gs[i].res_type, gs[i].relation, gs[i].subj_type, gs[i].subj_rel = s.add(g.rt), s.add(g.rel), s.add(g.st), s.add(g.srel)
		gs[i].res_ids = (*C.char)(C.CBytes(append(g.res, 0)))
		gs[i].subj_ids = (*C.char)(C.CBytes(append(g.subj, 0)))
		gs[i].res_off = (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&g.roff[0])), len(g.roff)*4)))
		gs[i].subj_off = (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&g.soff[0])), len(g.soff)*4)))
		s.p = append(s.p, unsafe.Pointer(gs[i].res_ids), unsafe.Pointer(gs[i].subj_ids), unsafe.Pointer(gs[i].res_off),
			unsafe.Pointer(gs[i].subj_off))
		if g.expiring {
			gs[i].expires_at = (*C.uint32_t)(C.CBytes(unsafe.Slice((*byte)(unsafe.Pointer(&g.exp[0])), len(g.exp)*4)))
			s.p = append(s.p, unsafe.Pointer(gs[i].expires_at))
		}
		gs[i].n = C.uint64_t(len(g.exp))
	}
	var n C.uint64_t
	return call(func() C.int { return C.zg_import_relationships(c.engine, arr, C.uint64_t(len(order)), &n) })
}

// RetireUnusedNames frees the interned names that no relationship of the mirror and no retained watch change mentions
// any more, and returns how many; later names reuse their ids, so the id space stays flat under the proxy's churn.
// The shim passes only strings and holds no ids, so nothing it caches goes stale. Run it right after CollectExpired.
func (c *Client) RetireUnusedNames() (uint64, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var n C.uint64_t
	if err := call(func() C.int { return C.zg_retire_unused_names(c.engine, &n) }); err != nil {
		return 0, err
	}
	return uint64(n), nil
}

// MirrorPage is one page of ReadMirrorPage: the lines ("type:id#rel@stype:sid[#srel]") in the page order, each line's
// expiration (zero time: none) and the cursor that resumes after it, the cursor after the page, and whether more follow.
type MirrorPage struct {
	Lines   []string
	Expires []time.Time
	Cursors [][]byte
	Next    []byte
	More    bool
}

// ReadMirrorPage reads the first `limit` relationships of the mirror that match the filter and follow `after` (nil:
// from the start), in the page order (resource type, resource, relation class, subject). A cursor stays valid across
// writes; one from another filter is refused. It reads the mirror only: ReadRelationships keeps delegating to SpiceDB.
func (c *Client) ReadMirrorPage(filter *v1.RelationshipFilter, limit uint64, after []byte) (*MirrorPage, error) {
	var s cstrs
	defer s.free()
	var f C.zg_filter_ex
	s.fillFilterEx(&f, filter)
	var cur *C.zg_read_cursor
	if after != nil {
		if len(after) != C.ZG_READ_CURSOR_BYTES {
			return nil, status.Errorf(codes.InvalidArgument, "read cursor of %d bytes", len(after))
		}
		cur = (*C.zg_read_cursor)(C.CBytes(after))
		defer C.free(unsafe.Pointer(cur))
	}
	if limit > 1<<16 { // a page returns at most this many lines: More reports the rest
		limit = 1 << 16
	}
	for capBytes := uint64(1 << 16); ; {
		buf := C.malloc(C.size_t(capBytes))
		exp := make([]C.uint32_t, limit+1)
		curs := make([]C.zg_read_cursor, limit+1)
		var need C.size_t
		var n C.uint64_t
		var next C.zg_read_cursor
		var more C.int32_t
		big := false
		err := call(func() C.int {
			rc := C.zg_read_relationships_page_ex(c.engine, &f, C.uint64_t(limit), cur, (*C.char)(buf), C.size_t(capBytes), &need,
				&n, &exp[0], &curs[0], &next, &more)
			big = rc == C.ZG_E2BIG
			if big {
				return 0
			}
			return rc
		})
		if err != nil || big {
			C.free(buf)
			if err != nil {
				return nil, err
			}
			capBytes = uint64(need) + 16
			continue
		}
		p := &MirrorPage{More: more != 0, Next: C.GoBytes(unsafe.Pointer(&next), C.ZG_READ_CURSOR_BYTES)}
		text := C.GoString((*C.char)(buf))
		C.free(buf)
		if text != "" {
			p.Lines = strings.Split(strings.TrimSuffix(text, "\n"), "\n")
		}
		for i := range p.Lines {
			p.Cursors = append(p.Cursors, C.GoBytes(unsafe.Pointer(&curs[i]), C.ZG_READ_CURSOR_BYTES))
			if exp[i] != 0 {
				p.Expires = append(p.Expires, time.Unix(int64(exp[i]), 0))
			} else {
				p.Expires = append(p.Expires, time.Time{})
			}
		}
		return p, nil
	}
}

// DeleteMirrorLimited deletes from the mirror what DeleteRelationships with optional_limit and
// optional_allow_partial_deletions deletes: more than `limit` matches fail with FailedPrecondition unless allowPartial,
// which deletes the first `limit` in the page order and reports partial. limit 0 deletes every match. The shim's
// DeleteRelationships keeps delegating to SpiceDB and mirroring the whole filter.
func (c *Client) DeleteMirrorLimited(filter *v1.RelationshipFilter, limit uint64, allowPartial bool) (uint64, bool, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var s cstrs
	defer s.free()
	var f C.zg_filter_ex
	s.fillFilterEx(&f, filter)
	var n C.uint64_t
	var partial C.int32_t
	allow := C.int(0)
	if allowPartial {
		allow = 1
	}
	if err := call(func() C.int {
		return C.zg_delete_relationships_limited_ex(c.engine, &f, nil, 0, C.uint64_t(limit), allow, &n, &partial)
	}); err != nil {
		return 0, false, err
	}
	return uint64(n), partial != 0, nil
}

// resync rebuilds the mirror from a full ReadRelationships per resource type. The mirror is EMPTIED
// first: it runs when a mirrored write failed after SpiceDB committed, and a batch that was rejected as a
// whole may have carried DELETEs -- re-TOUCHing what SpiceDB holds now would leave those revoked grants
// in place (fail-open). Until the rebuilt snapshot is published nothing is visible: zg_clear_relationships
// publishes the empty store, so a check that races the rebuild is denied, not wrongly allowed.
func (c *Client) resync(ctx context.Context) error {
	if err := call(func() C.int { return C.zg_clear_relationships(c.engine) }); err != nil {
		return err
	}
	nTypes := int(C.zg_num_types(c.engine))
	for t := 0; t < nTypes; t++ {
		typeName := C.GoString(C.zg_type_name(c.engine, C.int(t)))
		stream, err := c.PermissionsServiceClient.ReadRelationships(ctx, &v1.ReadRelationshipsRequest{
			Consistency:        &v1.Consistency{Requirement: &v1.Consistency_FullyConsistent{FullyConsistent: true}},
			RelationshipFilter: &v1.RelationshipFilter{ResourceType: typeName},
		})
		if err != nil {
			return err
		}
		var batch []*v1.RelationshipUpdate
		flush := func() error {
			if len(batch) == 0 {
				return nil
			}
			err := c.mirror(batch)
			batch = batch[:0]
			return err
		}
		for {
			r, err := stream.Recv()
			if err == io.EOF {
				break
			}
			if err != nil {
				return err
			}
			batch = append(batch, &v1.RelationshipUpdate{Operation: v1.RelationshipUpdate_OPERATION_TOUCH, Relationship: r.GetRelationship()})
			if len(batch) == 1000 { // pkg/spicedb/spicedb.go:34 WithMaximumUpdatesPerWrite(1000)
				if err := flush(); err != nil {
					return err
				}
			}
		}
		if err := flush(); err != nil {
			return err
		}
	}
	if err := call(func() C.int { return C.zg_publish(c.engine) }); err != nil {
		return err
	}
	c.broken.Store(false)
	return nil
}

// ListTemplate is the standard post-filter template, "T:{{namespacedName}}#perm@S:subject"
// (or {{name}}), with its literal fields already resolved for this request.
type ListTemplate struct {
	ResourceType, Permission                string
	SubjectType, SubjectID, SubjectRelation string
	RequestName, RequestNamespace           string // fallbacks of rules.NewResolveInput (pkg/rules/rules.go:321-326)
	NameOnly                                bool   // {{name}} instead of {{namespacedName}}
	ClearNamespace                          bool   // the request is on `namespaces` (rules.go:331-333)
}

// FilterListResponse replaces the body of filterListResponse (pkg/authz/postfilter.go:17-55) for rules whose
// PostFilters are all standard templates: one structural scan of the body, one bulk check on the GPU, one
// splice of the kept items -- no map[string]interface{} round trip, no per-item strings across cgo.
// The result is the same JSON value the reference produces (unknown fields, key order and number spelling
// are the apiserver's, since nothing is re-serialised).
func (c *Client) FilterListResponse(body []byte, tpls []ListTemplate) ([]byte, error) {
	if len(body) == 0 {
		return nil, fmt.Errorf("failed to parse list response: empty body")
	}
	var cs cstrs
	defer cs.free()
	ct := make([]C.zg_list_template, len(tpls))
	for i, t := range tpls {
		ct[i] = C.zg_list_template{
			res_type: cs.add(t.ResourceType), permission: cs.add(t.Permission),
			subj_type: cs.add(t.SubjectType), subj_id: cs.add(t.SubjectID), subj_rel: cs.add(t.SubjectRelation),
			req_name: cs.add(t.RequestName), req_namespace: cs.add(t.RequestNamespace),
			id_kind: C.ZG_ID_NAMESPACED_NAME,
		}
		if t.NameOnly {
			ct[i].id_kind = C.ZG_ID_NAME
		}
		if t.ClearNamespace {
			ct[i].flags = C.ZG_TPL_CLEAR_NAMESPACE
		}
	}
	var tp *C.zg_list_template
	if len(ct) > 0 {
		tp = &ct[0]
	}
	out := make([]byte, len(body)+8) // the filtered body is never longer than body + 2
	var outLen C.size_t
	if c.broken.Load() {
		return nil, errBroken
	}
	if err := call(func() C.int {
		return C.zg_list_postfilter(c.engine, (*C.char)(unsafe.Pointer(&body[0])), C.size_t(len(body)), tp, C.uint32_t(len(ct)),
			(*C.char)(unsafe.Pointer(&out[0])), C.size_t(len(out)), &outLen)
	}); err != nil {
		return nil, fmt.Errorf("failed to filter items with bulk permissions: %w", err)
	}
	return out[:outLen], nil
}

// PrefilterListResponse replaces runLookupResources + filterList / filterTable (pkg/authz/lookups.go:44-132,
// pkg/authz/responsefilterer.go:349-400) for rules whose pre-filter is the usual "namespace/name" split: one
// LookupResources on the GPU (concurrent list requests share launches), one scan of the body, one splice.
// contentType is the response's Content-Type header: kube clients get protobuf for built-in types and the reference
// decodes with the serializer it names (responsefilterer.go:241-266); asTable = the request's Accept carried
// "as=Table" (always JSON, responsefilterer.go:344-346).
func (c *Client) PrefilterListResponse(body []byte, contentType string, asTable bool, t ListTemplate) ([]byte, error) {
	if len(body) == 0 {
		return nil, fmt.Errorf("failed to decode response body: empty body")
	}
	mode := C.uint32_t(C.ZG_LIST_ITEMS)
	switch {
	case asTable:
		mode = C.ZG_LIST_TABLE_ROWS
	case strings.HasPrefix(strings.TrimSpace(contentType), "application/vnd.kubernetes.protobuf"):
		mode = C.ZG_LIST_PROTOBUF
	}
	var cs cstrs
	defer cs.free()
	ct := C.zg_list_template{
		res_type: cs.add(t.ResourceType), permission: cs.add(t.Permission),
		subj_type: cs.add(t.SubjectType), subj_id: cs.add(t.SubjectID), subj_rel: cs.add(t.SubjectRelation),
		req_name: cs.add(t.RequestName), req_namespace: cs.add(t.RequestNamespace),
	}
	out := make([]byte, len(body)+8)
	var outLen C.size_t
	if c.broken.Load() {
		return nil, errBroken
	}
	if err := call(func() C.int {
		return C.zg_list_prefilter(c.engine, (*C.char)(unsafe.Pointer(&body[0])), C.size_t(len(body)), mode, &ct,
			(*C.char)(unsafe.Pointer(&out[0])), C.size_t(len(out)), &outLen)
	}); err != nil {
		return nil, fmt.Errorf("failed to filter response: %w", err)
	}
	return out[:outLen], nil
}

var _ v1.PermissionsServiceClient = (*Client)(nil)
var _ = fmt.Sprintf
