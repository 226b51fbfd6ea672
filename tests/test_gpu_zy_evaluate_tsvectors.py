"""GPU, large: bm25x_evaluate_tsvectors where its casts run in several chunks and its kernel over millions of pairs, bit
for bit against bm25x_evaluate_batch over the four-step route (every pair) and the oracle over the restated casts (a
sample of pairs):
- a document batch of more than 2^22 entries and a query batch whose lexeme areas pass 64 MiB (util_tsvector's
  byte-cut batch), both cut into several cast chunks;
- one call of more than 2·10^6 pairs, every pair against one query.
Batches above 2^32 elements, which the 64-bit row offsets are for, are too large to build here and are untested."""
import numpy as np
import pytest

from util_documents import segment
from util_evaluate_tsvector import SEED, _bm, four_step, oracle_pairs
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_tsvector import (CHUNK_BYTES, CHUNK_ENT, assemble, byte_cut_batch, cast, cast_cuts, pack_ids, synthetic,
                           word_table)

pytestmark = pytest.mark.gpu


def _oracle(m, orc, tsv, k1=1.2, b=0.75):
    off, keys, tf = cast(_bm(m).intern, SEED, tsv)
    s = segment(off, tf, elem_key=keys)
    return s, orc.OracleIndex(orc.Corpus(s.n_docs, s.doc_len, s.n_terms, s.post_off, s.post_doc, s.post_tf, k1, b))


def _sample(m, oix, s, docs, queries, pair_query, got, rng, n=3000):
    """The oracle's evaluate of n sampled pairs (their documents taken out of the batch) against got."""
    pick = np.unique(rng.integers(0, len(docs["ent_off"]) - 1, n))
    ent, byt = docs["ent_off"].astype(np.int64), docs["byte_off"].astype(np.int64)
    sub = assemble([(docs["data"][byt[p]:byt[p + 1]], docs["entries"][ent[p]:ent[p + 1]]) for p in pick])
    d_off, dt, dtf, q_off, qt = oracle_pairs(m, s.term_keys, s.n_terms, sub, queries, np.asarray(pair_query)[pick])
    sel = lambda off, flat, i: flat[int(off[i]):int(off[i + 1])]
    want = np.array([oix.evaluate(sel(d_off, dt, i), sel(d_off, dtf, i), sel(q_off, qt, i)) for i in range(len(pick))])
    assert np.array_equal(got[pick], want)


def test_chunked_documents_and_queries(m, orc):
    rng = np.random.default_rng(1)
    tsv, words, _ = synthetic(rng, 20_000, 20, 80, 6000, 0.2)
    ix = m.Index.from_tsvectors(SEED, **tsv)
    s, oix = _oracle(m, orc, tsv)
    # documents: 50 000 tsvectors of 60..140 entries over the index's words and 2 000 more
    flat, off = word_table(words + [b"unknown-%d" % i for i in range(2000)])
    lens = rng.integers(60, 141, 50_000)
    wid = rng.integers(0, len(words) + 2000, int(lens.sum()))
    docs = pack_ids(lens, flat, off, wid, rng.integers(1, 5, len(wid)))
    assert int(docs["ent_off"][-1]) > CHUNK_ENT and len(cast_cuts(docs)) >= 2
    # queries: areas of about 1 MiB past 64 MiB in all, plus tsvectors of the index's words
    big, bwords, _ = byte_cut_batch()
    assert int(big["byte_off"][-1]) > CHUNK_BYTES and len(cast_cuts(big)) >= 2
    qlens = rng.integers(1, 8, 2000)
    small = pack_ids(qlens, flat, off, rng.integers(0, len(words), int(qlens.sum())), np.full(int(qlens.sum()), -1))
    nb = len(big["ent_off"]) - 1
    queries = dict(ent_off=np.concatenate([big["ent_off"], small["ent_off"][1:] + big["ent_off"][-1]]),
                   entries=np.concatenate([big["entries"], small["entries"]]),
                   byte_off=np.concatenate([big["byte_off"], small["byte_off"][1:] + big["byte_off"][-1]]),
                   data=np.concatenate([big["data"], small["data"]]))
    pq = rng.integers(nb, nb + 2000, 50_000).astype(np.uint32)
    pq[::97] = rng.integers(0, nb, len(pq[::97]))
    got = ix.evaluate_tsvectors(SEED, docs, queries, pq)
    assert np.array_equal(got, four_step(m, ix, docs, queries, pq))
    assert np.count_nonzero(got) > 1000
    _sample(m, oix, s, docs, queries, pq, got, rng)
    ix.close()


def test_two_million_pairs_in_one_call(m, orc):
    rng = np.random.default_rng(2)
    tsv, words, _ = synthetic(rng, 5000, 5, 30, 3000, 0.1)
    ix = m.Index.from_tsvectors(SEED, **tsv)
    s, oix = _oracle(m, orc, tsv)
    flat, off = word_table(words)
    n = 2_100_000
    lens = rng.integers(0, 5, n)
    wid = rng.integers(0, 300, int(lens.sum()))
    docs = pack_ids(lens, flat, off, wid, rng.integers(1, 4, len(wid)))
    one = pack_ids([10], flat, off, np.arange(0, 300, 30), np.full(10, -1))
    pq = np.zeros(n, np.uint32)
    got = ix.evaluate_tsvectors(SEED, docs, one, pq)
    assert len(got) == n and np.count_nonzero(got) > n // 20
    assert np.array_equal(got, four_step(m, ix, docs, one, pq))
    _sample(m, oix, s, docs, one, pq, got, rng)
    ix.close()
