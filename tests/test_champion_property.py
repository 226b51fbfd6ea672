"""The property the seeded kernel rests on (DESIGN.md §4.1 "seeds", §5), checked on the CPU with the oracle alone:

    a document that holds exactly ONE term of a query and belongs to the query's top-k is among the first k
    "champions" of that term — the term's postings in result order (exact single-term score desc, doc id asc),

so a query may take its single-term documents from the first min(k, df) champions of its terms and its stream needs to
find only the documents that two of its terms hold.  (The GPU side of it: tests/test_gpu_parity.py,
test_kernel_paths_identical — seeded launches return the bits of the unseeded kernel.)"""
import numpy as np
import pytest


@pytest.mark.parametrize("cfg", [
    dict(seed=61, n=4000, vocab=300, lmin=8, lmax=8, zipf=0.0),      # constant length: whole lists tie on the score
    dict(seed=62, n=6000, vocab=900, lmin=1, lmax=120, zipf=0.0),    # varied lengths
    dict(seed=63, n=5000, vocab=1500, lmin=10, lmax=60, zipf=1.0),   # Zipf: head terms, tf > 1
])
def test_single_holder_results_are_champions(orc, cfg):
    c = orc.Corpus.synth(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"])
    ix = orc.OracleIndex(c)
    q_off, q_terms = orc.gen_queries(cfg["seed"] + 1000, 80, cfg["vocab"], 2, 6, ix.df, cfg["zipf"])
    post_off, post_doc = np.asarray(c.post_off), np.asarray(c.post_doc)
    holders_of = {}
    champions = {}

    def docs_of(t):
        if t not in holders_of:
            holders_of[t] = set(int(d) for d in post_doc[post_off[t]:post_off[t + 1]])
        return holders_of[t]

    def champs(t):  # a single-term query ranks exactly in champion order: (score desc, doc asc)
        if t not in champions:
            champions[t] = [int(d) for d in ix.search_exhaustive([t], ix.df(int(t)))[0]]
        return champions[t]

    checked = 0
    for k in (1, 3, 10, 40):
        for i in range(len(q_off) - 1):
            q = [int(t) for t in q_terms[q_off[i]:q_off[i + 1]]]
            od, _, _ = ix.search_exhaustive(q, k)
            for d in od:
                held = [t for t in q if int(d) in docs_of(t)]
                assert held, "a result holds at least one query term"
                if len(held) == 1:
                    assert int(d) in champs(held[0])[:k], (cfg["seed"], i, k, int(d), held[0])
                    checked += 1
    assert checked > 50   # the property was actually exercised


def test_restated_champion_lists_are_single_term_rankings(orc):
    """The champion lists of the CPU restatement the GPU index tests compare with (tests/util_index.py) are each term's
    single-term ranking by the oracle, cut to min(df, 128) — with whole tie groups at the cut (b = 0) and without."""
    from util_index import restate
    for b, cfg in ((0.75, (62, 6000, 900, 1, 120, 0.0)), (0.0, (61, 4000, 100, 8, 8, 0.0))):
        c = orc.Corpus.synth(*cfg, b=b)
        ix = orc.OracleIndex(c)
        r = restate(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, c.k1, b, doc_len=c.doc_len)
        champ = r.champ.reshape(-1, 2)
        cut = 0
        for t in range(c.n_terms):
            lo, hi = int(r.champ_off[t]), int(r.champ_off[t + 1])
            od, os_, _ = ix.search_exhaustive([t], 129)
            assert np.array_equal(champ[lo:hi, 0], od[:128]), (b, t)
            p0, p1 = int(c.post_off[t]), int(c.post_off[t + 1])
            tf = c.post_tf[p0:p1][np.searchsorted(c.post_doc[p0:p1], od[:128])]
            assert np.array_equal(champ[lo:hi, 1] >> 8, tf), (b, t)
            cut += len(os_) > 128 and os_[127] == os_[128]
        assert cut > (20 if b == 0 else -1), cut
