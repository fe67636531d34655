"""LookupResources pages without a GPU: the cursor checks of zg_lookup_resources_page (a cursor is checked before the
engine's kind, so a host-only engine refuses a bad one with ZG_EINVAL and reaches the device refusal with a good one),
the refusals of host-only engines with the unpaged call's codes and messages, the client.py mirror's response cursors
over an engine stub, and the exported symbols."""
import struct

import pytest

EINVAL, ECUDA = -1, -4
SCHEMA = ("definition user {}\ndefinition doc {\n  relation viewer: user\n  relation editor: user\n"
          "  permission view = viewer + editor\n}\n")
LOOKUP_VERSION, READ_VERSION = 0x8001, 1


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _fnv(data, h=0xcbf29ce484222325):
    for b in data:
        h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def _fingerprint(rt, perm, st, srel, subj=None, name=None):
    """capi.cu lookup_fingerprint restated: a tag, the resolved ids and the form, then the subject as given."""
    h = _fnv(b"LookupResources")
    h = _fnv(struct.pack("<5H", rt, perm, st, srel, 1 if name is not None else 0), h)
    if name is not None:
        raw = name.encode()
        return _fnv(struct.pack("<Q", len(raw)) + raw, h)
    return _fnv(struct.pack("<I", subj), h)


def _cursor(version, has_key, gen, fp, rt=0, res=0):
    return struct.pack("<HHIQ4I", version, has_key, gen, fp, rt, res, 0, 0)


def _engine(zg):
    e = zg.Engine(SCHEMA, host_only=True)
    e.write_relationships([(0, "doc:a#viewer@user:u", 0), (0, "doc:b#editor@user:u", 0)])
    return e


def _code(fn):
    try:
        fn()
    except Exception as x:  # ZgpuError
        return getattr(x, "code", None), str(x)
    return 0, ""


def _ids(e):
    return e.type_id("doc"), e.slot_id("doc", "view"), e.type_id("user"), 0xFFFF


def test_cursor_checks_before_the_engine_kind(zg):
    e = _engine(zg)
    rt, perm, st, srel = _ids(e)
    u = e.find("user", "u")
    gen = None
    for g in range(4):  # the schema generation is not exported: the cursor that passes names it
        c = _cursor(LOOKUP_VERSION, 1, g, _fingerprint(rt, perm, st, srel, subj=u), rt, 0)
        if _code(lambda: e.lookup_resources_page("doc", "view", "user", u, limit=2, after=c))[0] == ECUDA:
            gen = g
    assert gen is not None, "no restated lookup cursor passed the checks"
    good = _cursor(LOOKUP_VERSION, 1, gen, _fingerprint(rt, perm, st, srel, subj=u), rt, 0)
    page = lambda after, subj=u, limit=2: _code(lambda: e.lookup_resources_page("doc", "view", "user", subj, limit=limit,  # noqa: E731
                                                                               after=after))
    assert page(None)[0] == ECUDA and page(good)[0] == ECUDA
    bad = {
        "another subject": _cursor(LOOKUP_VERSION, 1, gen, _fingerprint(rt, perm, st, srel, subj=u + 1), rt, 0),
        "another permission": _cursor(LOOKUP_VERSION, 1, gen, _fingerprint(rt, e.slot_id("doc", "viewer"), st, srel, subj=u)),
        "the string form": _cursor(LOOKUP_VERSION, 1, gen, _fingerprint(rt, perm, st, srel, name="u"), rt, 0),
        "a read cursor": _cursor(READ_VERSION, 1, gen, _fingerprint(rt, perm, st, srel, subj=u), rt, 0),
        "past the ids in the id form": _cursor(LOOKUP_VERSION, 2, gen, _fingerprint(rt, perm, st, srel, subj=u)),
        "another schema generation": _cursor(LOOKUP_VERSION, 1, gen + 1, _fingerprint(rt, perm, st, srel, subj=u), rt, 0),
        "zeros": bytes(32),
    }
    for why, c in bad.items():
        code, msg = page(c)
        assert code == EINVAL and "lookup cursor" in msg, why
    # a real read cursor of this engine (host-only engines page reads from the host store)
    read_next = e.read_relationships_page(1, None, res_type="doc")[3]
    assert page(read_next)[0] == EINVAL
    assert page(None, limit=0)[0] == EINVAL


def test_host_only_refusals_match_the_unpaged_call(zg):
    e = _engine(zg)
    u = e.find("user", "u")
    whole = _code(lambda: e.lookup_resources_ids("doc", "view", "user", u))
    assert whole[0] == ECUDA
    assert _code(lambda: e.lookup_resources_page("doc", "view", "user", u, limit=3)) == whole
    s_whole = _code(lambda: e.lookup_resources_str("doc", "view", "user", "u"))
    assert s_whole[0] == ECUDA
    assert _code(lambda: e.lookup_resources_page_str("doc", "view", "user", "u", limit=3)) == s_whole
    assert _code(lambda: e.lookup_resources_page_str("doc", "view", "user", "u", limit=0))[0] == EINVAL
    assert _code(lambda: e.lookup_page_counters()) == (0, "")
    assert e.lookup_page_counters() == {"windowed_pages": 0, "cut_pages": 0, "after_cursor": 0, "verified": 0, "windows": 0}


class _PagedStub:
    """lookup_resources_page_str over a fixed answer, with cursors that name the position after each name."""

    def __init__(self, names):
        self.names, self.calls = names, []

    def lookup_resources_page_str(self, rt, perm, st, sid, srel, limit, after):
        self.calls.append((limit, after))
        start = 0 if after is None else int.from_bytes(after, "little")
        page = self.names[start:start + limit]
        curs = [(start + i + 1).to_bytes(32, "little") for i in range(len(page))]
        return page, curs, curs[-1] if curs else (after or bytes(32)), start + limit < len(self.names)

    def lookup_resources_str(self, *q):
        return list(self.names)


def test_client_mirror_response_cursors_resume_the_rest(zg):
    from spicedb_kubeapi_proxy_b200 import client as cl

    names = [f"d{i}" for i in range(2500)]
    stub = _PagedStub(names)
    c = cl.PermissionsClient.__new__(cl.PermissionsClient)
    c.engine = stub
    subj = cl.SubjectReference(cl.ObjectReference("user", "u"))
    req = lambda **kw: cl.LookupResourcesRequest("doc", "view", subj, **kw)  # noqa: E731
    # neither: the unpaged call, no cursors
    plain = list(c.LookupResources(req()))
    assert [r.resource_object_id for r in plain] == names and all(r.after_result_cursor is None for r in plain)
    # a limit: one page of at most the limit
    page = list(c.LookupResources(req(optional_limit=7)))
    assert [r.resource_object_id for r in page] == names[:7]
    # only a cursor: every page after it; resuming from any response's cursor gives the rest
    rest = list(c.LookupResources(req(optional_cursor=page[3].after_result_cursor)))
    assert [r.resource_object_id for r in rest] == names[4:]
    for k in (0, 999, 1000, 2494):
        more = list(c.LookupResources(req(optional_cursor=rest[k].after_result_cursor)))
        assert [r.resource_object_id for r in more] == names[5 + k:]


def test_new_symbols_are_exported(zg):
    from spicedb_kubeapi_proxy_b200 import _lib

    L = _lib.lib()
    for name in ("zg_lookup_resources_page", "zg_lookup_resources_page_str", "zg_lookup_page_counters"):
        assert hasattr(L, name), name
    for m in ("lookup_resources_page", "lookup_resources_page_str", "iter_lookup_resources", "lookup_page_counters"):
        assert callable(getattr(zg.Engine, m)), m
