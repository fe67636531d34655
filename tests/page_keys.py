"""The page order of zg_read_relationships_page restated from a schema's text, for the suites that check it: the key
K = (resource type id, resource id, class position, subject id). A relation's classes are its allowed subject kinds in
the order the schema lists them, and a type's relations follow each other in the order they are declared, so the class
position is the index of (relation, subject type, subject relation) in that sequence. A wildcard's subject id is 0."""
from __future__ import annotations

import re


def class_positions(schema: str) -> dict:
    """{(resource type, relation, subject type, subject relation or "" or "*"): class position}."""
    out = {}
    for tname, body in re.findall(r"definition\s+(\w+)\s*\{(.*?)\}", schema, re.S):
        pos = 0
        for rel, expr in re.findall(r"relation\s+(\w+)\s*:\s*(.*?)(?=\brelation\b|\bpermission\b|$)", body, re.S):
            for term in expr.split("|"):
                term = re.sub(r"\bwith\s+expiration\b", "", term).strip()
                if term.endswith(":*"):
                    st, sr = term[:-2], "*"
                else:
                    st, _, sr = term.partition("#")
                out[(tname, rel, st.strip(), sr.strip())] = pos
                pos += 1
    return out


def page_key(e, positions: dict, line: str):
    """K of a relationship line, with ids from e.type_id / e.find."""
    left, right = line.split("@", 1)
    rt, rest = left.split(":", 1)
    rid, rel = rest.rsplit("#", 1)
    st, srest = right.split(":", 1)
    sid, _, srel = srest.partition("#")
    wild = sid == "*"
    return (e.type_id(rt), e.find(rt, rid), positions[(rt, rel, st, "*" if wild else srel)], 0 if wild else e.find(st, sid))
