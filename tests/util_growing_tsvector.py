"""The twin of a growing segment fed tsvectors (bm25x_growing_insert_tsvectors): a second segment on the same sealed
side fed bm25x_growing_insert with the restated rows (the host cast over bm25x_intern, the sealed lookup, fresh keys
numbered n_terms + K + rank in key order, each row re-sorted by ordinal), and the comparisons of a segment and of a seal
with the twin's, bit for bit."""
import numpy as np

from util_index import DERIVED, LAYOUT, fieldnorms, read_back
from util_parity import same_rows
from util_tsvector import cast

SEED = bytes((5 * i + 11) & 0xFF for i in range(32))
KS = (1, 10, 128, 1025)
MISSING = 0xFFFFFFFF


def bm_of(m):
    return __import__(m.__name__ + ".bm25x", fromlist=["x"])


class Twin:
    """The restated inserts on a second segment over the same sealed side."""

    def __init__(self, m, sealed):
        self.m, self.sealed, self.T = m, sealed, sealed.n_terms
        self.seg = sealed.growing_segment()
        self.keys = {}                      # key bytes -> ordinal, for the keys the sealed vocabulary lacks

    def rows(self, tsv):
        off, keys, tf = cast(bm_of(self.m).intern, SEED, tsv)
        n = len(off) - 1
        ords = self.sealed.lookup_terms(keys) if len(keys) else np.zeros(0, np.uint32)
        miss = np.nonzero(ords == MISSING)[0]
        fresh = sorted({bytes(keys[i]) for i in miss} - set(self.keys))
        new = {k: self.T + len(self.keys) + r for r, k in enumerate(fresh)}
        for i in miss:
            k = bytes(keys[i])
            ords[i] = self.keys[k] if k in self.keys else new[k]
        vec = np.repeat(np.arange(n), np.diff(off.astype(np.int64)))
        order = np.lexsort((ords, vec))
        lens = np.bincount(vec, weights=tf.astype(np.float64), minlength=n) if len(vec) else np.zeros(n)
        return off, ords[order], tf[order], np.minimum(lens, 0xFFFFFFFF).astype(np.uint32), new

    def insert(self, orc, tsv, payload=None, form="doc_len"):
        off, ords, tf, lens, new = self.rows(tsv)
        norm = dict(doc_len=lens) if form == "doc_len" else dict(doc_fieldnorm=fieldnorms(orc, lens))
        self.seg.insert(off, ords, tf, payload=payload, **norm)
        self.keys.update(new)

    def new_keys(self):
        out = np.zeros((len(self.keys), 16), np.uint8)
        for k, t in self.keys.items():
            out[t - self.T] = np.frombuffer(k, np.uint8)
        return out


def same_arrays(lay_a, der_a, lay_b, der_b, what):
    a, b = read_back(lay_a, der_a), read_back(lay_b, der_b)
    for name, _ in LAYOUT + DERIVED:
        if (name in ("blk", "blk_ub") and lay_b.n_blocks == 0) or (name == "champ" and der_b.n_champ == 0):
            continue
        assert a[name].tobytes() == b[name].tobytes(), f"{what}: {name} differs"


def same_segment(seg, twin, queries, what):
    """Arrays, info, keys and search rows of seg equal the twin's."""
    assert np.array_equal(seg.new_keys(), twin.new_keys()), f"{what}: new keys"
    seg.refresh()
    twin.seg.refresh()
    a, b = seg.info(), twin.seg.info()
    for f, _ in type(b)._fields_:
        assert getattr(a, f) == getattr(b, f), f"{what}: info.{f}"
    if a.n_docs:
        same_arrays(*seg.arrays(), *twin.seg.arrays(), what)
    q_off, q_terms = seg.tsvector_queries(SEED, **queries)
    for k in KS:
        same_rows(seg.search_batch(q_off, q_terms, k, want_payload=True),
                  twin.seg.search_batch(q_off, q_terms, k, want_payload=True), f"{what} k={k}")


def same_seal(got, want, what):
    """Two seals: maps, info, and every handle's arrays (each shard's for a sharded index)."""
    ix_a, ix_b = got[0], want[0]
    for x, y, name in zip(got[1:], want[1:], ("sealed_map", "growing_map", "term_map")):
        assert np.array_equal(x, y), f"{what}: {name}"
    a, b = ix_a.info(), ix_b.info()
    for f, _ in type(b)._fields_:
        assert getattr(a, f) == getattr(b, f), f"{what}: info.{f}"
    if hasattr(ix_b, "shard_arrays"):
        assert np.array_equal(ix_a.doc_bounds(), ix_b.doc_bounds()), what
        for s in range(len(ix_b.doc_bounds()) - 1):
            same_arrays(*ix_a.shard_arrays(s), *ix_b.shard_arrays(s), f"{what} shard {s}")
    else:
        same_arrays(ix_a.layout(), ix_a.derived(), ix_b.layout(), ix_b.derived(), what)
    rng = np.random.default_rng(3)
    T = a.n_terms
    qs = [rng.choice(T, size=min(T, int(rng.integers(1, 6))), replace=False) for _ in range(40)]
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    q_terms = np.array([t for q in qs for t in q], np.uint32)
    for k in KS:
        same_rows(ix_a.search_batch(q_off, q_terms, k, want_payload=True),
                  ix_b.search_batch(q_off, q_terms, k, want_payload=True), f"{what} sealed k={k}")
