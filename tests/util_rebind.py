"""The restatement of a rebind (bm25x_growing_rebind) on the CPU: the carried documents of a growing segment as the one
insert into a fresh segment over the seal's result that the rebound segment equals, and the late deletes."""
from types import SimpleNamespace

import numpy as np

from util_index import ctid
from util_maintain import MISSING

NONE = 0xFFFFFFFF


class Refused(Exception):
    """The rebind refuses the carried documents (a keyed caller-numbered ordinal without a new ordinal)."""


def restate(docs, n_folded, kind, *, term_map=None, old_keys=None, seg_keys=None, new_keys=None, new_n_terms=0):
    """docs: every old ordinal's document (elem_off, elem_term, elem_tf, deleted flags now, payload [n, 3] or None,
    doc_len or doc_fieldnorm, either None).  kind: "keyless", "owned" (keys: old_keys of the old sealed terms, seg_keys of
    the segment's own, new_keys of the new index, which has new_n_terms terms) or "caller" (the seal's term_map).
    Returns the carried documents as bm25x_growing_insert takes them (ordinal n_folded + i as document i) and, owned,
    the keys the segment numbers after the rebind.  A deleted carried document keeps no element."""
    off = np.asarray(docs.elem_off, np.int64)
    n = len(off) - 1
    to_old = len(old_keys) if old_keys is not None else 0
    new_ord = {bytes(k): i for i, k in enumerate(np.asarray(new_keys, np.uint8).reshape(-1, 16))} if kind == "owned" else {}

    def key_of(t):
        return bytes(old_keys[t]) if t < to_old else bytes(seg_keys[t - to_old])

    rows = []   # per carried document: [(old term, tf)]
    for o in range(n_folded, n):
        if docs.deleted[o]:
            rows.append([])
            continue
        rows.append([(int(t), int(f)) for t, f in zip(docs.elem_term[off[o]:off[o + 1]], docs.elem_tf[off[o]:off[o + 1]])])
    lack = sorted({key_of(t) for r in rows for t, _ in r if t != MISSING and kind == "owned" and key_of(t) not in new_ord})
    fresh = {k: new_n_terms + i for i, k in enumerate(lack)}

    def translate(o, t):
        if t == MISSING or kind == "keyless":
            return t
        if kind == "owned":
            k = key_of(t)
            return new_ord[k] if k in new_ord else fresh[k]
        if t >= len(term_map):
            raise Refused(f"growing ordinal {o} holds term ordinal {t} >= n_source_terms={len(term_map)}")
        if term_map[t] == MISSING:
            raise Refused(f"growing ordinal {o} holds term ordinal {t}, whose key vanished in the seal")
        return int(term_map[t])

    e_off, e_term, e_tf = [0], [], []
    for i, r in enumerate(rows):
        el = sorted((translate(n_folded + i, t), f) for t, f in r)
        e_term += [t for t, _ in el]
        e_tf += [f for _, f in el]
        e_off.append(len(e_term))
    c = slice(n_folded, n)
    payload = np.asarray(docs.payload, np.uint16)[c] if docs.payload is not None else ctid(np.arange(n_folded, n))
    return SimpleNamespace(
        elem_off=np.array(e_off, np.uint64), elem_term=np.array(e_term, np.uint32), elem_tf=np.array(e_tf, np.uint32),
        deleted=np.asarray(docs.deleted, np.uint8)[c].copy(), payload=payload.reshape(-1, 3),
        doc_len=None if docs.doc_len is None else np.asarray(docs.doc_len, np.uint32)[c],
        doc_fieldnorm=None if docs.doc_fieldnorm is None else np.asarray(docs.doc_fieldnorm, np.uint8)[c],
        owned_keys=np.array([np.frombuffer(k, np.uint8) for k in lack], np.uint8).reshape(-1, 16))


def late_deleted(growing_map, deleted):
    """The new ids of the folded ordinals (those growing_map covers) deleted after the seal's snapshot, ascending."""
    gm = np.asarray(growing_map, np.uint32)
    d = np.asarray(deleted[:len(gm)], bool)
    return np.sort(gm[d & (gm != NONE)]).astype(np.uint32)


def insert_kw(r):
    """bm25x_growing_insert arguments of a restatement."""
    kw = dict(elem_off=r.elem_off, elem_term=r.elem_term, elem_tf=r.elem_tf, deleted=r.deleted, payload=r.payload)
    if r.doc_len is not None:
        kw["doc_len"] = r.doc_len
    else:
        kw["doc_fieldnorm"] = r.doc_fieldnorm
    return kw
