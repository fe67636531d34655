"""PermissionsClient -- host-side mirror of the reference's drop-in boundary.

The reference holds a `v1.PermissionsServiceClient` (authzed-go v1.6.0) in
`Options.PermissionsClient` (pkg/proxy/options.go:81-82,371-377) and calls exactly
these methods on it:

    CheckBulkPermissions   pkg/authz/check.go:48, pkg/authz/postfilter.go:134
    CheckPermission        pkg/authz/watch.go:50
    LookupResources        pkg/authz/lookups.go:65  (server stream until io.EOF)
    LookupSubjects         (v1 API; in the client mock of pkg/authz/postfilter_test.go:71, no call site)
    Watch                  pkg/authz/watch.go:29   (v1.WatchServiceClient, same connection)
    WriteRelationships     pkg/authz/distributedtx/activity.go:60
    ReadRelationships      pkg/authz/distributedtx/activity.go:107,154
    DeleteRelationships    (v1 API; the proxy deletes by read-then-write, workflow.go:354-389)
    ExpandPermissionTree   (v1 API; debugging tools: `zed permission expand`)

Same method names, same request/response field names and the same error behaviour
(per-pair errors inside a successful bulk response; a failed precondition fails the
whole write), so the parity tests read like the reference's own. In a Go build the
same role is played by the cgo shim in go/gpuauthz (INTEGRATION.md); here, with no
Go toolchain, this Python class drives the identical C ABI.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Iterable, Iterator, List, Optional

from . import _lib
from ._lib import Engine, ZgpuError

# v1.CheckPermissionResponse_Permissionship
PERMISSIONSHIP_UNSPECIFIED = 0
PERMISSIONSHIP_NO_PERMISSION = 1
PERMISSIONSHIP_HAS_PERMISSION = 2
PERMISSIONSHIP_CONDITIONAL_PERMISSION = 3
# v1.LookupPermissionship
LOOKUP_PERMISSIONSHIP_HAS_PERMISSION = 1
# v1.LookupSubjectsRequest_WildcardOption
WILDCARD_OPTION_UNSPECIFIED, WILDCARD_OPTION_INCLUDE_WILDCARDS, WILDCARD_OPTION_EXCLUDE_WILDCARDS = 0, 1, 2
# v1.AlgebraicSubjectSet_Operation
OPERATION_UNSPECIFIED, OPERATION_UNION, OPERATION_INTERSECTION, OPERATION_EXCLUSION = 0, 1, 2, 3
# v1.RelationshipUpdate_Operation
OPERATION_CREATE, OPERATION_TOUCH, OPERATION_DELETE = 1, 2, 3
# v1.Precondition_Operation
PRECONDITION_MUST_NOT_MATCH, PRECONDITION_MUST_MATCH = 1, 2

_OP = {OPERATION_CREATE: _lib.OP_CREATE, OPERATION_TOUCH: _lib.OP_TOUCH, OPERATION_DELETE: _lib.OP_DELETE}
_PRE = {PRECONDITION_MUST_MATCH: _lib.PRECOND_MUST_MATCH, PRECONDITION_MUST_NOT_MATCH: _lib.PRECOND_MUST_NOT_MATCH}


@dataclass
class ObjectReference:
    object_type: str
    object_id: str


@dataclass
class SubjectReference:
    object: ObjectReference
    optional_relation: str = ""


@dataclass
class Relationship:
    resource: ObjectReference
    relation: str
    subject: SubjectReference
    optional_expires_at: int = 0  # unix seconds, 0 = none

    def text(self) -> str:
        s = f"{self.resource.object_type}:{self.resource.object_id}#{self.relation}@" \
            f"{self.subject.object.object_type}:{self.subject.object.object_id}"
        return s + (f"#{self.subject.optional_relation}" if self.subject.optional_relation else "")

    @staticmethod
    def parse(rel: str, expires_at: int = 0) -> "Relationship":
        rt, rid, r, st, sid, srel = _lib.split_rel(rel)
        return Relationship(ObjectReference(rt, rid), r, SubjectReference(ObjectReference(st, sid), srel), expires_at)


@dataclass
class CheckBulkPermissionsRequestItem:
    resource: ObjectReference
    permission: str
    subject: SubjectReference


@dataclass
class CheckBulkPermissionsRequest:
    items: List[CheckBulkPermissionsRequestItem]
    fully_consistent: bool = True  # every call site in the reference sets FullyConsistent


@dataclass
class CheckBulkPermissionsResponseItem:
    permissionship: int


@dataclass
class CheckBulkPermissionsPair:
    request: CheckBulkPermissionsRequestItem
    item: Optional[CheckBulkPermissionsResponseItem] = None
    error: Optional[str] = None  # google.rpc.Status message

    def GetError(self):
        return self.error

    def GetItem(self):
        return self.item


@dataclass
class CheckBulkPermissionsResponse:
    pairs: List[CheckBulkPermissionsPair]


@dataclass
class CheckPermissionRequest:
    resource: ObjectReference
    permission: str
    subject: SubjectReference
    fully_consistent: bool = True


@dataclass
class CheckPermissionResponse:
    permissionship: int


@dataclass
class LookupResourcesRequest:
    resource_object_type: str
    permission: str
    subject: SubjectReference
    fully_consistent: bool = True
    optional_limit: int = 0  # 0: no limit
    optional_cursor: Optional[bytes] = None  # an after_result_cursor of an earlier response


@dataclass
class LookupResourcesResponse:
    resource_object_id: str
    permissionship: int = LOOKUP_PERMISSIONSHIP_HAS_PERMISSION
    after_result_cursor: Optional[bytes] = None  # set when the request had a limit or a cursor


@dataclass
class LookupSubjectsRequest:
    resource: ObjectReference
    permission: str
    subject_object_type: str
    optional_subject_relation: str = ""
    wildcard_option: int = WILDCARD_OPTION_UNSPECIFIED
    fully_consistent: bool = True


@dataclass
class ResolvedSubject:
    subject_object_id: str  # "*" for the wildcard
    permissionship: int = LOOKUP_PERMISSIONSHIP_HAS_PERMISSION


@dataclass
class LookupSubjectsResponse:
    subject: ResolvedSubject
    excluded_subjects: List[ResolvedSubject] = field(default_factory=list)  # only on the wildcard


@dataclass
class ExpandPermissionTreeRequest:
    resource: ObjectReference
    permission: str
    fully_consistent: bool = True


@dataclass
class DirectSubjectSet:
    subjects: List[SubjectReference]


@dataclass
class AlgebraicSubjectSet:
    operation: int
    children: List["PermissionRelationshipTree"]


@dataclass
class PermissionRelationshipTree:
    expanded_object: ObjectReference
    expanded_relation: str
    intermediate: Optional[AlgebraicSubjectSet] = None  # exactly one of intermediate and leaf is set
    leaf: Optional[DirectSubjectSet] = None


@dataclass
class ExpandPermissionTreeResponse:
    tree_root: PermissionRelationshipTree


_EXPAND_OP = {"U": OPERATION_UNION, "I": OPERATION_INTERSECTION, "X": OPERATION_EXCLUSION}


def _expand_tree(n: dict) -> PermissionRelationshipTree:
    obj = ObjectReference(*n["object"].split(":", 1))
    if n["op"] == "L":
        subjects = []
        for x in n["subjects"]:
            t, rest = x.split(":", 1)
            sid, _, srel = rest.partition("#")
            subjects.append(SubjectReference(ObjectReference(t, sid), srel))
        return PermissionRelationshipTree(obj, n["relation"], leaf=DirectSubjectSet(subjects))
    return PermissionRelationshipTree(obj, n["relation"], intermediate=AlgebraicSubjectSet(
        _EXPAND_OP[n["op"]], [_expand_tree(c) for c in n["children"]]))


@dataclass
class RelationshipUpdate:
    operation: int
    relationship: Relationship


@dataclass
class SubjectFilter:
    subject_type: str
    optional_subject_id: str = ""
    optional_relation: str = ""  # v1 wraps this in SubjectFilter_RelationFilter


@dataclass
class RelationshipFilter:
    resource_type: str = ""
    optional_resource_id: str = ""
    optional_relation: str = ""
    optional_subject_filter: Optional[SubjectFilter] = None
    # only relationships whose resource's id starts with it (every resource type when resource_type is empty)
    optional_resource_id_prefix: str = ""

    def fields(self) -> dict:
        f = {"res_type": self.resource_type, "res_id": self.optional_resource_id, "rel": self.optional_relation}
        if self.optional_resource_id_prefix:
            f["res_id_prefix"] = self.optional_resource_id_prefix
        if self.optional_subject_filter:
            s = self.optional_subject_filter
            f.update(subj_type=s.subject_type, subj_id=s.optional_subject_id, subj_rel=s.optional_relation)
        return f


@dataclass
class Precondition:
    operation: int
    filter: RelationshipFilter


@dataclass
class WriteRelationshipsRequest:
    updates: List[RelationshipUpdate]
    optional_preconditions: List[Precondition] = field(default_factory=list)


@dataclass
class WriteRelationshipsResponse:
    written_at: int  # snapshot revision that contains the write


@dataclass
class DeleteRelationshipsRequest:
    relationship_filter: RelationshipFilter
    optional_preconditions: List[Precondition] = field(default_factory=list)
    optional_limit: int = 0  # 0: every match
    optional_allow_partial_deletions: bool = False


DELETION_PROGRESS_COMPLETE, DELETION_PROGRESS_PARTIAL = 1, 2  # v1.DeleteRelationshipsResponse_DeletionProgress


class DeleteRelationshipsResponse(int):
    """The number of relationships deleted (what DeleteRelationships always returned), carrying deletion_progress."""

    deletion_progress: int = DELETION_PROGRESS_COMPLETE

    def __new__(cls, deleted: int, deletion_progress: int = DELETION_PROGRESS_COMPLETE):
        r = super().__new__(cls, deleted)
        r.deletion_progress = deletion_progress
        return r


@dataclass
class ReadRelationshipsRequest:
    relationship_filter: RelationshipFilter
    fully_consistent: bool = True
    optional_limit: int = 0  # 0: no limit
    optional_cursor: Optional[bytes] = None  # an after_result_cursor of an earlier response


@dataclass
class ReadRelationshipsResponse:
    relationship: Relationship
    after_result_cursor: Optional[bytes] = None  # set when the request had a limit or a cursor


@dataclass
class ExportBulkRelationshipsRequest:
    optional_limit: int = 0  # relationships per response; 0: 1 000
    optional_cursor: Optional[bytes] = None


@dataclass
class ExportBulkRelationshipsResponse:
    after_result_cursor: bytes
    relationships: List[Relationship]


@dataclass
class ImportBulkRelationshipsRequest:
    relationships: List[Relationship]


@dataclass
class ImportBulkRelationshipsResponse:
    num_loaded: int


@dataclass
class WatchRequest:
    optional_object_types: List[str] = field(default_factory=list)
    optional_start_cursor: Optional[int] = None  # revision; None = changes after the call (watch.go:29-31)


@dataclass
class WatchResponse:
    updates: List[RelationshipUpdate]
    changes_through: int  # revision; usable as the next optional_start_cursor


class RpcError(Exception):
    """Stands in for a gRPC status error (codes follow google.rpc.Code names)."""

    def __init__(self, code: str, message: str):
        super().__init__(f"{code}: {message}")
        self.code = code
        self.message = message


def _rpc(e: ZgpuError) -> RpcError:
    code = {-1: "INVALID_ARGUMENT", -2: "ALREADY_EXISTS", -3: "FAILED_PRECONDITION", -5: "FAILED_PRECONDITION",
            -6: "FAILED_PRECONDITION", -8: "RESOURCE_EXHAUSTED"}.get(e.code, "INTERNAL")
    return RpcError(code, str(e))


class PermissionsClient:
    """Implements the v1.PermissionsServiceClient methods the proxy calls, on the GPU."""

    def __init__(self, schema: str, relationships=(), device: int = -1, engine: Engine | None = None):
        self.engine = engine or Engine(schema, device=device)
        if relationships:
            self.WriteRelationships(WriteRelationshipsRequest(
                [RelationshipUpdate(OPERATION_TOUCH, Relationship.parse(r)) for r in relationships]))

    # -- checks -----------------------------------------------------------------
    def CheckBulkPermissions(self, req: CheckBulkPermissionsRequest) -> CheckBulkPermissionsResponse:
        rels = [(it.resource.object_type, it.resource.object_id, it.permission, it.subject.object.object_type,
                 it.subject.object.object_id, it.subject.optional_relation) for it in req.items]
        try:
            codes = self.engine.check_bulk_str(rels)
        except ZgpuError as e:
            raise _rpc(e) from None
        pairs = []
        for it, c in zip(req.items, codes):  # pairs[i] answers items[i] (pkg/authz/check.go:54-57)
            if c == _lib.ITEM_ERROR:
                pairs.append(CheckBulkPermissionsPair(it, error="check failed: unknown permission/type or max depth exceeded"))
            else:
                pairs.append(CheckBulkPermissionsPair(it, item=CheckBulkPermissionsResponseItem(int(c))))
        return CheckBulkPermissionsResponse(pairs)

    def CheckPermission(self, req: CheckPermissionRequest) -> CheckPermissionResponse:
        resp = self.CheckBulkPermissions(CheckBulkPermissionsRequest(
            [CheckBulkPermissionsRequestItem(req.resource, req.permission, req.subject)]))
        pair = resp.pairs[0]
        if pair.error:
            raise RpcError("FAILED_PRECONDITION", pair.error)
        return CheckPermissionResponse(pair.item.permissionship)

    def LookupResources(self, req: LookupResourcesRequest) -> Iterator[LookupResourcesResponse]:
        """Slice-backed stand-in for the server stream (pkg/authz/lookups.go:74-88). Without a limit or a cursor: the
        unpaged answer. With a limit: one page of at most optional_limit resources after the cursor; with only a
        cursor: every resource after it. Resources come in ascending interned id order, each with the cursor that
        resumes after it."""
        q = (req.resource_object_type, req.permission, req.subject.object.object_type, req.subject.object.object_id,
             req.subject.optional_relation)
        try:
            if not req.optional_limit and req.optional_cursor is None:
                return iter([LookupResourcesResponse(i) for i in self.engine.lookup_resources_str(*q)])
            out, cursor = [], req.optional_cursor
            while True:
                names, curs, cursor, more = self.engine.lookup_resources_page_str(*q, limit=req.optional_limit or 1000,
                                                                                  after=cursor)
                out += [LookupResourcesResponse(n, after_result_cursor=c) for n, c in zip(names, curs)]
                if not more or req.optional_limit:
                    return iter(out)
        except ZgpuError as e:
            raise _rpc(e) from None

    def LookupSubjects(self, req: LookupSubjectsRequest) -> Iterator[LookupSubjectsResponse]:
        """Slice-backed stand-in for the server stream: the concrete subjects, then (when a wildcard grants the
        permission and the option includes wildcards) `*` with the subjects it excludes."""
        opt = _lib.WILDCARDS_EXCLUDE if req.wildcard_option == WILDCARD_OPTION_EXCLUDE_WILDCARDS else _lib.WILDCARDS_INCLUDE
        try:
            ids, wild, excluded = self.engine.lookup_subjects_str(req.resource.object_type, req.resource.object_id,
                                                                  req.permission, req.subject_object_type,
                                                                  req.optional_subject_relation, opt)
        except ZgpuError as e:
            raise _rpc(e) from None
        out = [LookupSubjectsResponse(ResolvedSubject(i)) for i in ids]
        if wild:
            out.append(LookupSubjectsResponse(ResolvedSubject("*"), [ResolvedSubject(x) for x in excluded]))
        return iter(out)

    def ExpandPermissionTree(self, req: ExpandPermissionTreeRequest) -> ExpandPermissionTreeResponse:
        """The permission's subject tree at the resource, one level of usersets deep (v1's shallow expansion): leaves
        list the relationships' subjects, arrows expand into the subtrees of their targets."""
        try:
            lines = self.engine.expand_permission_tree_str(req.resource.object_type, req.resource.object_id, req.permission)
        except ZgpuError as e:
            raise _rpc(e) from None
        return ExpandPermissionTreeResponse(_expand_tree(_lib.parse_expand_lines(lines)))

    # -- relationships ------------------------------------------------------------
    def WriteRelationships(self, req: WriteRelationshipsRequest) -> WriteRelationshipsResponse:
        ups = [(_OP[u.operation], u.relationship.text(), u.relationship.optional_expires_at) for u in req.updates]
        pre = [(_PRE[p.operation], p.filter.fields()) for p in req.optional_preconditions]
        try:
            self.engine.write_relationships(ups, pre)
        except ZgpuError as e:
            raise _rpc(e) from None
        return WriteRelationshipsResponse(self.engine.stats()["revision"])

    def DeleteRelationships(self, req: DeleteRelationshipsRequest) -> DeleteRelationshipsResponse:
        pre = [(_PRE[p.operation], p.filter.fields()) for p in req.optional_preconditions]
        try:
            if not req.optional_limit:
                return DeleteRelationshipsResponse(self.engine.delete_relationships(req.relationship_filter.fields(), pre))
            n, partial = self.engine.delete_relationships_limited(req.relationship_filter.fields(), pre, req.optional_limit,
                                                                  req.optional_allow_partial_deletions)
        except ZgpuError as e:
            raise _rpc(e) from None
        return DeleteRelationshipsResponse(n, DELETION_PROGRESS_PARTIAL if partial else DELETION_PROGRESS_COMPLETE)

    def Watch(self, req: WatchRequest) -> "WatchStream":
        """v1.WatchServiceClient.Watch (pkg/authz/watch.go:27-48). The returned stream is polled:
        `Recv()` hands back the next WatchResponse (one per revision, as SpiceDB groups updates by
        transaction) or None when the feed is drained -- the gRPC stream would block instead."""
        for t in req.optional_object_types:
            if self.engine.type_id(t) < 0:
                raise RpcError("INVALID_ARGUMENT", f"object definition `{t}` not found")
        start = req.optional_start_cursor
        if start is None:
            start = self.engine.stats()["revision"]
        return WatchStream(self.engine, list(req.optional_object_types), start)

    def ReadRelationships(self, req: ReadRelationshipsRequest) -> Iterator[ReadRelationshipsResponse]:
        """Without a limit or a cursor: the unpaged read, sorted. With them: the matches after the cursor in the page
        order (at most optional_limit of them), each with its expiration and the cursor that resumes after it."""
        flt = req.relationship_filter.fields()
        try:
            if not req.optional_limit and req.optional_cursor is None:
                lines = self.engine.read_relationships(**flt)
                return iter([ReadRelationshipsResponse(Relationship.parse(l)) for l in lines])
            out, cursor, left = [], req.optional_cursor, req.optional_limit
            while True:
                lines, exp, curs, cursor, more = self.engine.read_relationships_page(min(left, 1000) if left else 1000,
                                                                                    cursor, **flt)
                out += [ReadRelationshipsResponse(Relationship.parse(l, x), c) for l, x, c in zip(lines, exp, curs)]
                if req.optional_limit:
                    left -= len(lines)
                if not more or (req.optional_limit and left == 0):
                    return iter(out)
        except ZgpuError as e:
            raise _rpc(e) from None

    def ExportBulkRelationships(self, req: ExportBulkRelationshipsRequest) -> Iterator[ExportBulkRelationshipsResponse]:
        """Every relationship after the cursor, in the page order, optional_limit per response (the empty filter)."""
        out, cursor = [], req.optional_cursor
        try:
            while True:
                lines, exp, _, cursor, more = self.engine.read_relationships_page(req.optional_limit or 1000, cursor)
                if lines:
                    out.append(ExportBulkRelationshipsResponse(cursor, [Relationship.parse(l, x) for l, x in zip(lines, exp)]))
                if not more:
                    return iter(out)
        except ZgpuError as e:
            raise _rpc(e) from None

    def ImportBulkRelationships(self, requests: Iterable[ImportBulkRelationshipsRequest]) -> ImportBulkRelationshipsResponse:
        """The client stream of ImportBulkRelationships: every request's relationships are CREATEs of one transaction,
        imported all-or-nothing and published once. They are grouped by class (first appearance of the class, then
        the order given), and new names get their ids in that order. The `relationship <i>` of an error message counts
        in that grouped order too; it equals the stream's order when each class's relationships arrive together."""
        rels = [(r.text(), r.optional_expires_at) for req in requests for r in req.relationships]
        try:
            n = self.engine.import_relationships(self.engine.import_groups(rels))
        except ZgpuError as e:
            raise _rpc(e) from None
        return ImportBulkRelationshipsResponse(n)


_WATCH_OP = {"TOUCH": OPERATION_TOUCH, "CREATE": OPERATION_CREATE, "DELETE": OPERATION_DELETE}


class WatchStream:
    def __init__(self, engine: Engine, object_types: List[str], cursor: int):
        self.engine, self.object_types, self.cursor = engine, object_types, cursor
        self._pending: List[WatchResponse] = []

    def _fill(self):
        try:
            if len(self.object_types) == 1:
                changes, through = self.engine.watch_read(self.cursor, self.object_types[0])
            else:
                changes, through = self.engine.watch_read(self.cursor, "")
                if self.object_types:
                    keep = tuple(t + ":" for t in self.object_types)
                    changes = [c for c in changes if c[2].startswith(keep)]
        except ZgpuError as e:
            raise _rpc(e) from None
        by_rev: dict = {}
        for rev, op, rel, exp in changes:
            by_rev.setdefault(rev, []).append(RelationshipUpdate(_WATCH_OP[op], Relationship.parse(rel, exp)))
        self._pending = [WatchResponse(ups, rev) for rev, ups in sorted(by_rev.items())]
        self.cursor = through

    def Recv(self) -> Optional[WatchResponse]:
        if not self._pending:
            self._fill()
        return self._pending.pop(0) if self._pending else None

    def __iter__(self):
        while True:
            r = self.Recv()
            if r is None:
                return
            yield r
