"""numpy restatement of the reference's seal, `maintain` (crates/bm25/src/maintain.rs:27-311): the corpus of the new
sealed segment from the sealed one, the sealed deleted set and the growing documents.  Data movement only: the scoring
arithmetic stays in the C oracle (util_index.restate, OracleIndex).

What it follows:
- maintain.rs:56-73, add_document (330-342): the sealed documents in id order; a deleted one gets no record, a surviving
  one the next record id, with its stored payload and length 0.
- maintain.rs:104-158, add_element (344-362): every posting of a surviving sealed document is written under the new id
  and adds 1 to the record's length (saturating_add(1)): a sealed survivor's length is its number of postings, not Σ tf.
- maintain.rs:167-255: then the growing documents in chain order; a deleted one is skipped, a surviving one goes through
  io::write with Document::new(elements): its length is Document::length, the saturating Σ tf of ALL its elements
  (vector.rs:77-83), unknown tokens included; given as doc_len when the caller stored exact lengths.
- flush (maintain.rs:263-266): tokens with at least one mapping, ascending key; N = records, Σlen = Σ lengths.
Token identities: a sealed term is its key (keyed index) or its ordinal (keyless); a growing element names a source
ordinal: < n_terms(sealed) a sealed term, beyond it ordinal n_terms(sealed) + i with key new_keys[i] (keyed) or itself
(keyless, where every ordinal up to the largest inserted stays a term, with df 0 when it has no posting);
TERM_MISSING never becomes a term."""
from types import SimpleNamespace

import numpy as np

from util_index import ctid

MISSING = 0xFFFFFFFF
U32_MAX = 0xFFFFFFFF


def maintain(n_docs, post_off, post_doc, post_tf, growing, *, sealed_deleted=None, sealed_payload=None, sealed_keys=None,
             new_keys=None):
    """n_docs / post_off / post_doc / post_tf: the sealed corpus (term-major CSR); growing: namespace of elem_off,
    elem_term, elem_tf, deleted (per ordinal), doc_len (None: doc_fieldnorm form) and payload (None: the synthetic ctid of
    the ordinal); sealed_deleted: bool per sealed id (None: none); sealed_payload: [n_docs, 3] (None: the synthetic ctid of
    the old id); sealed_keys: [n_terms, 16] (None: keyless); new_keys: [n, 16].  Returns the new corpus (n_docs, n_terms,
    post_off, post_doc, post_tf, doc_len, payload [n, 3], term_keys or None) and sealed_map, growing_map, term_map."""
    NS = int(n_docs)
    off = np.asarray(post_off, np.int64)
    T = len(off) - 1
    sdoc = np.asarray(post_doc, np.int64)
    stf = np.asarray(post_tf, np.int64)
    sdel = np.zeros(NS, bool) if sealed_deleted is None else np.asarray(sealed_deleted, bool)
    # records: sealed survivors first (ascending old id), growing survivors after them (ascending ordinal)
    smap = np.full(NS, U32_MAX, np.int64)
    smap[~sdel] = np.arange(int((~sdel).sum()))
    NSK = int((~sdel).sum())
    goff = np.asarray(growing.elem_off, np.int64)
    G = len(goff) - 1
    gdel = np.asarray(growing.deleted, bool) if growing.deleted is not None else np.zeros(G, bool)
    gmap = np.full(G, U32_MAX, np.int64)
    gmap[~gdel] = NSK + np.arange(int((~gdel).sum()))
    N = NSK + int((~gdel).sum())
    # add_element: the sealed survivors' postings, length += 1 each
    sterm = np.repeat(np.arange(T), np.diff(off))
    keep = ~sdel[sdoc]
    length = np.zeros(N, np.int64)
    length[:NSK] = np.bincount(smap[sdoc[keep]], minlength=NSK)[:NSK] if NSK else 0
    # io::write of the growing survivors: Document::length, or the stored exact length
    gterm = np.asarray(growing.elem_term, np.int64)
    gtf = np.asarray(growing.elem_tf, np.int64)
    gown = np.repeat(np.arange(G), np.diff(goff))
    if growing.doc_len is not None:
        glen = np.asarray(growing.doc_len, np.int64)
    else:
        glen = np.minimum(np.bincount(gown, weights=gtf, minlength=G).astype(np.int64) if G else np.zeros(0, np.int64),
                          U32_MAX)
    length[NSK:] = glen[~gdel]
    length = np.minimum(length, U32_MAX)
    # source terms
    known = gterm != MISSING
    if sealed_keys is not None:
        n_src = T + (0 if new_keys is None else len(new_keys))
        assert np.all(gterm[known] < n_src), "an inserted ordinal without a key"
    else:
        assert new_keys is None
        n_src = max(T, int(gterm[known].max()) + 1 if known.any() else 0)
    glive = known & ~gdel[gown]
    term = np.concatenate([sterm[keep], gterm[glive]])
    doc = np.concatenate([smap[sdoc[keep]], gmap[gown[glive]]])
    tf = np.concatenate([stf[keep], gtf[glive]])
    df_src = np.bincount(term, minlength=n_src)
    # flush: the tokens that have mappings, ascending key (keyless: every ordinal, df 0 included)
    if sealed_keys is not None:
        keys_all = np.concatenate([np.asarray(sealed_keys, np.uint8).reshape(-1, 16),
                                   np.asarray(new_keys if new_keys is not None else np.zeros((0, 16)), np.uint8).reshape(-1, 16)])
        src_of = sorted(np.flatnonzero(df_src > 0).tolist(), key=lambda t: keys_all[t].tobytes())
        src_of = np.array(src_of, np.int64)
        term_keys = keys_all[src_of] if len(src_of) else np.zeros((0, 16), np.uint8)
    else:
        src_of = np.arange(n_src)
        term_keys = None
    tmap = np.full(n_src, MISSING, np.int64)
    tmap[src_of] = np.arange(len(src_of))
    TN = len(src_of)
    nterm = tmap[term]
    order = np.lexsort((doc, nterm))
    new_off = np.concatenate([[0], np.cumsum(np.bincount(nterm, minlength=TN))]).astype(np.uint64)
    spay = ctid(np.arange(NS)) if sealed_payload is None else np.asarray(sealed_payload, np.uint16).reshape(-1, 3)
    gpay = ctid(np.arange(G)) if growing.payload is None else np.asarray(growing.payload, np.uint16).reshape(-1, 3)
    payload = np.concatenate([spay[~sdel], gpay[~gdel]]).astype(np.uint16)
    return SimpleNamespace(n_docs=N, n_terms=TN, post_off=new_off, post_doc=doc[order].astype(np.uint32),
                           post_tf=tf[order].astype(np.uint32), doc_len=length.astype(np.uint32), payload=payload,
                           term_keys=term_keys, sealed_map=smap.astype(np.uint32), growing_map=gmap.astype(np.uint32),
                           term_map=tmap.astype(np.uint32))
