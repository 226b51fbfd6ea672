"""GPU: the document-sharded index built from stored blocks (bm25x_index_create_sharded_from_blocks) against the sharded
index built from the decoded CSR (byte-identical arrays, shard by shard), against the CPU restatement of every shard
(tests/util_index.py), and against the unsharded stored-block ingest (bit-identical search rows on every kernel path, the
same refusals for every corruption, wherever it sits relative to the shard bounds)."""

import numpy as np
import pytest

from util_corpora import ADVERSARIAL_BOUNDS, BLOCK_CONFIGS, SHARDED_PATHS, adversarial_corpus
from util_cuda import free_bytes
from util_index import DERIVED, LAYOUT, SCALARS, assert_matches, check_shards, local_csr, read_back, restate
from util_lib import gpu_library, refused  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import query_csr, same_rows

pytestmark = pytest.mark.gpu


def _dict(c):
    """A synthetic corpus as a CSR dict of copies (its own arrays are views of memory the library frees with it)."""
    return dict(n_docs=c.n_docs, doc_len=c.doc_len.copy(), n_terms=c.n_terms, post_off=c.post_off.copy(),
                post_doc=c.post_doc.copy(), post_tf=c.post_tf.copy())


def _encode(orc, c):
    """(blocks kwargs of Index.from_blocks, EncodedBlocks) of a CSR dict."""
    eb = orc.EncodedBlocks(orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"],
                                      c["post_tf"]))
    return dict(n_docs=c["n_docs"], n_terms=c["n_terms"], term_blk_off=eb.term_blk_off, blk_min_doc=eb.blk_min,
                blk_n=eb.blk_n, blk_meta_doc=eb.meta_doc, blk_meta_tf=eb.meta_tf, blk_doc_off=eb.doc_off,
                blk_tf_off=eb.tf_off, data=eb.bytes[:eb.n_bytes], doc_len=c["doc_len"]), eb


def _same_shards(got, want, what):
    """Every shard's layout and derived arrays byte-identical (placeholder slots of empty arrays aside)."""
    assert np.array_equal(got.doc_bounds(), want.doc_bounds()), what
    b = want.doc_bounds()
    for s in range(len(b) - 1):
        (lg, dg), (lw, dw) = got.shard_arrays(s), want.shard_arrays(s)
        for name in SCALARS:
            assert getattr(lg, name) == getattr(lw, name), f"{what} shard {s}: {name}"
        assert dg.n_champ == dw.n_champ and dg.s1f_min == dw.s1f_min, f"{what} shard {s}"
        ag, aw = read_back(lg, dg), read_back(lw, dw)
        for name, _ in LAYOUT + DERIVED:
            if (name in ("blk", "blk_ub") and lw.n_blocks == 0) or (name == "champ" and dw.n_champ == 0):
                continue
            assert ag[name].tobytes() == aw[name].tobytes(), f"{what} shard {s} [{b[s]}, {b[s + 1]}): {name} differs"


def _same_info(sx, ix, what):
    a, w = sx.info(), ix.info()
    for f in ("n_docs", "n_terms", "n_postings", "sum_doc_len", "avgdl", "k1", "b", "device"):
        assert getattr(a, f) == getattr(w, f), (what, f)


def _rows(ix, sx, q_off, q_terms, k, allow=None, what=""):
    want = ix.search_batch(q_off, q_terms, k, allow=allow, want_payload=True)
    got = sx.search_batch(q_off, q_terms, k, allow=allow, want_payload=True)
    same_rows(got, want, what)


# ---- 1. arrays: byte-identical to bm25x_sharded_create on the decoded CSR ----

@pytest.mark.parametrize("cfg", BLOCK_CONFIGS, ids=[c["name"] for c in BLOCK_CONFIGS])
def test_arrays_identical_to_sharded_create(m, orc, cfg):
    c = _dict(m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"]))
    blocks, _ = _encode(orc, c)
    ix = m.Index.from_blocks(**blocks)
    rng = np.random.default_rng(cfg["seed"] & 0xFFFF)
    for S in (1, 2, 3, 16):
        explicit = np.r_[0, np.sort(rng.choice(np.arange(1, c["n_docs"]), S - 1, replace=False)), c["n_docs"]]
        for bounds in (None, explicit.astype(np.uint32)):
            what = f"{cfg['name']} S={S} bounds={'default' if bounds is None else bounds.tolist()}"
            want = m.ShardedIndex(**c, n_shards=S, doc_bounds=bounds)
            got = m.ShardedIndex.from_blocks(**blocks, n_shards=S, doc_bounds=bounds)
            _same_shards(got, want, what)
            _same_info(got, ix, what)
            assert got.info().device_bytes == want.info().device_bytes, what
            got.close()
            want.close()
    ix.close()


# ---- 2. bounds placed against the stored blocks ----

def _block_bounds(c, eb):
    """Bounds exactly at a stored block's first doc, at its last doc and last + 1, inside a full block and inside a
    byte-packed tail."""
    off, doc = c["post_off"].astype(np.int64), np.asarray(c["post_doc"])
    tbo = eb.term_blk_off.astype(np.int64)
    t = int(np.nonzero(np.diff(tbo) >= 3)[0][0])                  # a token with >= 3 blocks
    p = off[t] + 128                                                 # its second block, full
    tail_t = int(np.nonzero((np.diff(off) % 128 >= 20) & (np.diff(tbo) >= 1))[0][-1])
    q = off[tail_t + 1] - (np.diff(off)[tail_t] % 128) + 7          # inside the byte-packed tail of tail_t
    return sorted({0, int(doc[p]), int(doc[p + 127]), int(doc[p + 127]) + 1, int(doc[off[t] + 60]), int(doc[q]),
                   c["n_docs"]})


def test_bounds_against_blocks(m, orc):
    c = _dict(m.synth_corpus(22, 30000, 5000, 16, 96, 1.0))
    blocks, eb = _encode(orc, c)
    bounds = _block_bounds(c, eb)
    assert len(bounds) >= 6, bounds
    ix = m.Index(**c)
    sx = m.ShardedIndex.from_blocks(**blocks, n_shards=len(bounds) - 1, doc_bounds=bounds)
    check_shards(m, orc, c, sx, ix, 1.2, 0.75, f"block bounds {bounds}")
    want = m.ShardedIndex(**c, n_shards=len(bounds) - 1, doc_bounds=bounds)
    _same_shards(sx, want, "block bounds")
    q_off, q_terms = m.synth_queries(1022, 100, 5000, 1, 8, c["post_off"], 1.0)
    bix = m.Index.from_blocks(**blocks)
    for k in (10, 1000):
        _rows(bix, sx, q_off, q_terms, k, what=f"block bounds k={k}")
    for x in (sx, want, bix, ix):
        x.close()


def test_adversarial_bounds(m, orc):
    """A one-document shard, a shard with no postings at all, terms with no postings in some shards."""
    c, rng = adversarial_corpus()
    blocks, _ = _encode(orc, c)
    ix = m.Index(**c)
    sx = m.ShardedIndex.from_blocks(**blocks, n_shards=len(ADVERSARIAL_BOUNDS) - 1, doc_bounds=ADVERSARIAL_BOUNDS)
    check_shards(m, orc, c, sx, ix, 1.2, 0.75, "adversarial")
    bix = m.Index.from_blocks(**blocks)
    qs = [[60], [61], [60, 61], [60, 3, 7], [61, 5], [1, 2, 3, 4]]
    qs += [list(rng.choice(62, size=int(rng.integers(1, 9)), replace=False)) for _ in range(30)]
    q_off, q_terms = query_csr(qs)
    allow = np.packbits(rng.random(c["n_docs"]) < 0.4, bitorder="little")
    for k in (1, 100, 1025):
        for al in (None, allow):
            _rows(bix, sx, q_off, q_terms, k, allow=al, what=f"adversarial k={k}")
    for x in (sx, bix, ix):
        x.close()


# ---- 3. input variants ----

def test_stored_norms(m, orc):
    c = _dict(m.synth_corpus(41, 4000, 300, 4, 200, 0.7))
    blocks, _ = _encode(orc, c)
    fn = np.array([orc.lib().orc_length_to_fieldnorm(int(x)) for x in c["doc_len"]], dtype=np.uint8)
    total = int(c["doc_len"].astype(np.uint64).sum())
    stored = dict(blocks, doc_len=None, doc_fieldnorm=fn, sum_doc_len=total)
    ix = m.Index.from_blocks(**stored)
    bounds = [0, 999, 1000, 2500, 4000]
    sx = m.ShardedIndex.from_blocks(**stored, n_shards=4, doc_bounds=bounds)
    _same_info(sx, ix, "stored norms")
    off, doc, tf = c["post_off"], np.asarray(c["post_doc"]), np.asarray(c["post_tf"])
    stat = (c["n_docs"], np.diff(off.astype(np.int64)), total / c["n_docs"])
    for s in range(4):
        lo, hi = bounds[s], bounds[s + 1]
        lay, der = sx.shard_arrays(s)
        loff, ldoc, ltf = local_csr(off, doc, tf, lo, hi)
        r = restate(orc, hi - lo, loff, ldoc, ltf, 1.2, 0.75, fieldnorm=fn[lo:hi], sum_len=total, stat=stat, doc_base=lo)
        assert_matches(read_back(lay, der), lay, der, r, f"stored norms shard {s}")
    q_off, q_terms = m.synth_queries(42, 60, 300, 1, 6, off, 0.7)
    for k in (10, 129):
        _rows(ix, sx, q_off, q_terms, k, what=f"stored norms k={k}")
    sx2 = m.ShardedIndex.from_blocks(**stored, n_shards=3)   # default bounds from the decoded postings
    assert np.array_equal(sx2.doc_bounds(), m.ShardedIndex(**c, n_shards=3).doc_bounds())
    for x in (sx2, sx, ix):
        x.close()


def test_payload_and_term_keys(m, orc):
    c = _dict(m.synth_corpus(31, 3000, 100, 4, 40, 0.0))
    blocks, _ = _encode(orc, c)
    rng = np.random.default_rng(2)
    keys = np.unique(rng.integers(1, 255, size=(c["n_terms"] * 2, 16), dtype=np.uint8), axis=0)[:c["n_terms"]]
    payload = rng.integers(0, 65535, size=(c["n_docs"], 3)).astype(np.uint16)
    q_off, q_terms = m.synth_queries(32, 40, 100, 1, 4, c["post_off"])
    probe = np.concatenate([keys[::7], np.zeros((1, 16), np.uint8), keys[-1:]])
    for pl in (payload, None):
        ix = m.Index.from_blocks(**blocks, payload=pl, term_keys=keys)
        sx = m.ShardedIndex.from_blocks(**blocks, payload=pl, term_keys=keys, n_shards=3,
                                        doc_bounds=[0, 1001, 1999, c["n_docs"]])
        assert np.array_equal(sx.lookup_terms(probe), ix.lookup_terms(probe))
        for k in (3, 50):
            _rows(ix, sx, q_off, q_terms, k, what=f"payload={pl is not None} k={k}")
        sx.close()
        ix.close()


def _two_block_token(orc, docs, tfs, N):
    md0, pd0 = orc.compress_document_ids(int(docs[0]), docs[:128])
    mt0, pt0 = orc.compress_term_frequencies(tfs[:128])
    md1, pd1 = orc.compress_document_ids(int(docs[128]), docs[128:])
    mt1, pt1 = orc.compress_term_frequencies(tfs[128:])
    data = np.concatenate([pd0, pt0, pd1, pt1])
    offs = np.cumsum([0, len(pd0), len(pt0), len(pd1)])
    return dict(n_docs=N, n_terms=1, term_blk_off=[0, 2], blk_min_doc=[docs[0], docs[128]], blk_n=[128, len(docs) - 128],
                blk_meta_doc=[md0, md1], blk_meta_tf=[mt0, mt1], blk_doc_off=[offs[0], offs[2]],
                blk_tf_off=[offs[1], offs[3]], data=data, doc_fieldnorm=np.full(N, 20, dtype=np.uint8),
                sum_doc_len=20 * N), (md0, md1)


def test_wide_deltas_tf_limits_and_raw_tail(m, orc):
    """test_gpu_blocks.py's wide-delta / tf-limit blocks and its byte-width-4 raw tail, each cut by shard bounds."""
    N = 40_000_000
    rng = np.random.default_rng(5)
    docs = np.sort(rng.choice(N, 128 + 77, replace=False)).astype(np.uint32)
    docs[1] = docs[0] + 1
    tfs = rng.integers(1, 1 << 20, len(docs)).astype(np.uint32)
    tfs[3] = tfs[130] = (1 << 24) - 1
    blocks, (md0, _) = _two_block_token(orc, docs, tfs, N)
    assert md0 >> 7 == 0 and (md0 & 0x7F) >= 20
    bounds = [0, int(docs[2]), int(docs[60]) + 1, int(docs[140]), N]
    cases = [(blocks, bounds)]
    N2 = 60_000_000
    head = np.sort(rng.choice(1_000_000, 128, replace=False)).astype(np.uint32)
    first, second = 1_000_007, 1_000_007 + (1 << 24) + 5
    rest = np.sort(rng.choice(np.arange(second + 1, N2), 75, replace=False)).astype(np.uint32)
    docs2 = np.concatenate([head, [first, second], rest]).astype(np.uint32)
    blocks2, (_, md1) = _two_block_token(orc, docs2, rng.integers(1, 9, len(docs2)).astype(np.uint32), N2)
    assert md1 == (0x80 | 4)
    cases.append((blocks2, [0, first + 1, int(rest[40]), N2]))           # the raw tail cut twice
    for blk, b in cases:
        ix = m.Index.from_blocks(**blk)
        sx = m.ShardedIndex.from_blocks(**blk, n_shards=len(b) - 1, doc_bounds=b)
        for k in (1, 100, 1000):
            _rows(ix, sx, np.array([0, 1], np.uint32), np.array([0], np.uint32), k, what=f"bounds {b} k={k}")
        sx.close()
        ix.close()
    tfs[50] = 1 << 24
    blocks, _ = _two_block_token(orc, docs, tfs, N)
    want = refused(m, lambda: m.Index.from_blocks(**blocks))
    assert want[0] == 4 and "2^24" in want[1]
    assert refused(m, lambda: m.ShardedIndex.from_blocks(**blocks, n_shards=4, doc_bounds=bounds)) == want


# ---- 4. search rows on every kernel path ----

def test_search_every_path(m, orc):
    c = _dict(m.synth_corpus(81, 60000, 4000, 6, 40, 1.0))
    blocks, _ = _encode(orc, c)
    q_off, q_terms = m.synth_queries(82, 160, c["n_terms"], 1, 8, c["post_off"], 1.0)
    allow = np.packbits(np.random.default_rng(9).random(c["n_docs"]) < 0.5, bitorder="little")
    ix = m.Index.from_blocks(**blocks)
    sx = m.ShardedIndex.from_blocks(**blocks, n_shards=3)
    for name, opts in SHARDED_PATHS.items():
        for idx in (ix, sx):
            for o in ("seed", "twophase", "prune"):
                idx.set_option(o, {"seed": 1, "twophase": 0, "prune": 1}[o])
            idx.set_option("seed_dense_div", 64)
            idx.set_option("seed_prune_min", 32768)
            for o, v in opts.items():
                idx.set_option(o, v)
        for k in (1, 10, 100, 129, 1000):
            for al in (None, allow):
                _rows(ix, sx, q_off, q_terms, k, allow=al, what=f"{name} k={k} allow={al is not None}")
    sx.close()
    ix.close()


# ---- 5. corruption: the unsharded ingest's refusals, wherever the corrupt block sits ----

def _placements(doc_ids, N):
    """Bounds that cut the block holding doc_ids (ascending), and bounds whose last shard holds it whole."""
    a, z = int(doc_ids[0]), int(doc_ids[-1])
    assert 0 < a < z < N
    return {"straddles": [0, a + 1, N], "inside last shard": [0, a, N]}


def _same_refusal(m, blocks, doc_ids, what):
    want = refused(m, lambda: m.Index.from_blocks(**blocks))
    for where, b in _placements(doc_ids, blocks["n_docs"]).items():
        free = free_bytes()
        got = refused(m, lambda: m.ShardedIndex.from_blocks(**blocks, n_shards=2, doc_bounds=b))
        assert got == want, (what, where, got, want)
        assert free_bytes() == free, (what, where, "device memory not freed")
    return want


def test_corruption_matches_the_unsharded_ingest(m, orc):
    c = _dict(m.synth_corpus(43, 2000, 20, 8, 40, 0.5))
    blocks, eb = _encode(orc, c)
    m.ShardedIndex.from_blocks(**blocks, n_shards=2).close()          # every kernel loaded before memory is compared
    t2 = int(np.nonzero(np.diff(eb.term_blk_off.astype(np.int64)) >= 4)[0][0])
    full = int(eb.term_blk_off[t2]) + 1                               # a token's second block: full, not its last
    assert eb.blk_n[full] == 128 and eb.blk_n[full + 1] == 128
    o = int(c["post_off"][t2]) + 128
    ids = np.asarray(c["post_doc"])[o:o + 128]                        # the documents of block `full`
    cases = []
    bad = eb.blk_n.copy(); bad[full] = 100
    cases.append(("short block", dict(blocks, blk_n=bad)))
    bad = eb.meta_doc.copy(); bad[full] = 33
    cases.append(("bit width 33", dict(blocks, blk_meta_doc=bad)))
    bad = eb.doc_off.copy(); bad[full] = eb.n_bytes
    cases.append(("payload past the end", dict(blocks, blk_doc_off=bad)))
    bad = eb.blk_min.copy(); bad[full] = c["n_docs"]
    cases.append(("ids past n_docs", dict(blocks, blk_min_doc=bad)))
    data = blocks["data"].copy()
    w = int(eb.meta_tf[full]) & 0x7F
    data[int(eb.tf_off[full]):int(eb.tf_off[full]) + 16 * w] = 0
    cases.append(("tf 0", dict(blocks, data=data)))
    swap = lambda a: np.concatenate([a[:full], a[full + 1:full + 2], a[full:full + 1], a[full + 2:]])
    cases.append(("blocks out of order", dict(blocks, blk_min_doc=swap(eb.blk_min), blk_meta_doc=swap(eb.meta_doc),
                                               blk_meta_tf=swap(eb.meta_tf), blk_doc_off=swap(eb.doc_off),
                                               blk_tf_off=swap(eb.tf_off))))
    for what, blk in cases:
        code, msg = _same_refusal(m, blk, ids, what)
        assert code == 1 and "corrupt block" in msg, (what, msg)

    # a first delta that wraps past 2^32, in a full block and in a byte-packed tail
    N = 1000
    full_docs, tail_docs = 16 + 7 * np.arange(128, dtype=np.uint32), 16 + 5 * np.arange(50, dtype=np.uint32)
    md0, pd0 = orc.compress_document_ids(16, full_docs)
    md1, pd1 = orc.compress_document_ids(16, tail_docs)
    mt0, pt0 = orc.compress_term_frequencies(np.ones(128, np.uint32))
    mt1, pt1 = orc.compress_term_frequencies(np.ones(50, np.uint32))
    data = np.concatenate([pd0, pt0, pd1, pt1])
    offs = np.cumsum([0, len(pd0), len(pt0), len(pd1)])
    for mins in ((0xFFFFFFF0, 16), (16, 0xFFFFFFF0)):
        blk = dict(n_docs=N, n_terms=2, term_blk_off=[0, 1, 2], blk_min_doc=list(mins), blk_n=[128, 50],
                   blk_meta_doc=[md0, md1], blk_meta_tf=[mt0, mt1], blk_doc_off=[offs[0], offs[2]],
                   blk_tf_off=[offs[1], offs[3]], data=data, doc_fieldnorm=np.full(N, 20, dtype=np.uint8),
                   sum_doc_len=20 * N)
        code, msg = _same_refusal(m, blk, tail_docs, f"wrapped first delta {mins}")
        assert code == 1 and "corrupt blocks" in msg


def test_wand_corruption_matches_the_unsharded_ingest(m, orc):
    c = _dict(m.synth_corpus(47, 6000, 60, 4, 120, 0.9))
    blocks, eb = _encode(orc, c)
    oc = orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"])
    wfn, wtf = orc.OracleIndex(oc).block_wand()
    good = dict(blocks, blk_wand_fieldnorm=wfn, blk_wand_tf=wtf)
    ix = m.Index.from_blocks(**good)
    sx = m.ShardedIndex.from_blocks(**good, n_shards=3)
    _same_shards(sx, m.ShardedIndex(**c, n_shards=3), "wand given")
    sx.close()
    ix.close()
    tbo, off, doc = eb.term_blk_off.astype(np.int64), c["post_off"].astype(np.int64), np.asarray(c["post_doc"])

    def block_docs(g):
        t = int(np.searchsorted(tbo, g, side="right") - 1)
        a = off[t] + 128 * (g - tbo[t])
        return doc[a:min(a + 128, off[t + 1])]

    g = max((g for g in range(len(wtf)) if len(block_docs(g)) > 1 and block_docs(g)[0] > 0), key=lambda g: wtf[g])
    assert wtf[g] > 1                     # its arg-max has tf > 1: tf 1 lowers the bound
    bad_tf = wtf.copy()
    bad_tf[g] = 1
    code, msg = _same_refusal(m, dict(good, blk_wand_tf=bad_tf), block_docs(g), "wand tf")
    assert code == 1 and "wand" in msg
    g = next(g for g in range(len(wfn)) if len(block_docs(g)) > 1 and block_docs(g)[0] > 0)
    bad_fn = wfn.copy()
    bad_fn[g] = 255 if wfn[g] < 200 else 0
    code, msg = _same_refusal(m, dict(good, blk_wand_fieldnorm=bad_fn), block_docs(g), "wand fieldnorm")
    assert code == 1 and "wand" in msg


# ---- 6. two devices ----

def test_shards_on_two_devices(m, orc):
    if m.device_count() < 2:
        pytest.skip("one CUDA device visible: shards on two devices not exercised")
    c = _dict(m.synth_corpus(22, 30000, 5000, 16, 96, 1.0))
    blocks, _ = _encode(orc, c)
    q_off, q_terms = m.synth_queries(1022, 200, 5000, 1, 8, c["post_off"], 1.0)
    ix = m.Index.from_blocks(**blocks)
    sx = m.ShardedIndex.from_blocks(**blocks, n_shards=4, devices=[0, 1, 0, 1])
    allow = np.packbits(np.random.default_rng(1).random(c["n_docs"]) < 0.5, bitorder="little")
    for k in (10, 100, 1025):
        for al in (None, allow):
            _rows(ix, sx, q_off, q_terms, k, allow=al, what=f"two devices k={k}")
    sx.close()
    ix.close()
