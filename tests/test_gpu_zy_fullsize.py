"""BASELINE.json configs at their STATED size on the GPU (configs[2..4]): size-independent properties on the whole
batch (sortedness, canonical tie order, no document twice, pruning on/off identity) + a sample checked bit for bit
against the exhaustive oracle.  The corpora are the bench workloads (bench.py WORKLOADS: same seeds)."""
import numpy as np
import pytest

from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import oracle_index

pytestmark = pytest.mark.gpu


def _properties(res, k, n_docs, what):
    n = res["n"]
    s, d = res["score64"], res["doc"]
    cols = np.arange(k)[None, :]
    valid = cols < n[:, None]
    both = valid[:, 1:]                                      # pairs (i, i+1) that both exist
    assert np.all((s[:, :-1] >= s[:, 1:]) | ~both), f"{what}: not sorted by score"
    tie = (s[:, :-1] == s[:, 1:]) & both
    assert np.all(d[:, :-1][tie] < d[:, 1:][tie]), f"{what}: tie order is not ascending doc id"
    assert np.all(d[valid] < n_docs) and np.all(d[~valid] == 0xFFFFFFFF), f"{what}: doc ids out of range"
    assert np.all(s[valid] > 0.0)
    srt = np.sort(np.where(valid, d, np.arange(d.shape[1], dtype=np.uint64)[None, :] + (1 << 33)).astype(np.uint64), axis=1)
    assert np.all(srt[:, 1:] != srt[:, :-1]), f"{what}: a document appears twice in one result row"
    np.testing.assert_allclose(res["score"][valid], s[valid], rtol=1e-5, atol=0)


def _sample_vs_oracle(res, oix, q_off, q_terms, k, idx, what):
    for i in idx:
        q = q_terms[q_off[i]:q_off[i + 1]]
        od, os_, _ = oix.search_exhaustive(q, k)
        n = int(res["n"][i])
        assert n == len(od), f"{what} q{i}: n {n} != {len(od)}"
        assert np.array_equal(res["doc"][i, :n], od), f"{what} q{i} k{k}: ids\n got {res['doc'][i, :n]}\nwant {od}"
        assert np.array_equal(res["score64"][i, :n], os_), f"{what} q{i}: f64 scores not bit-exact"


def test_config3_full_100k_queries_top100_and_top10(m, orc):
    """configs[2]: 10M docs, vocab 100k, 128 terms/doc, 100k 3-term queries, top-100 (and the metric's top-10)."""
    c = m.synth_corpus(0xB25C0DE3, 10_000_000, 100_000, 128)
    q_off, q_terms = m.synth_queries(0xB25C0DE3 + 1000, 100_000, 100_000, 3, 3, c.post_off)
    ix = m.Index.from_corpus(c)
    oix = oracle_index(orc, c)
    for k in (100, 10):
        res = ix.search_batch(q_off, q_terms, k)
        assert np.all(res["n"] == k)
        _properties(res, k, c.n_docs, f"C3 k={k}")
        _sample_vs_oracle(res, oix, q_off, q_terms, k, range(0, 100_000, 1999), f"C3 k={k}")       # 51 queries
    ix.close()


def test_config4_zipf_8term_pruning_on_off(m, orc):
    """configs[3]: 10M docs, Zipf(1) term frequencies, 8-term queries, pruning on/off.  Pruning ON runs the whole
    100k-query batch; OFF (exhaustive: head terms have df → N, ≈ 240 MB of postings per query) runs the first 2000
    queries, on which both must agree bit for bit."""
    c = m.synth_corpus(0xB25C0DE4, 10_000_000, 100_000, 128, 128, 1.0)
    q_off, q_terms = m.synth_queries(0xB25C0DE4 + 1000, 100_000, 100_000, 8, 8, c.post_off, 1.0)
    ix = m.Index.from_corpus(c)
    on = ix.search_batch(q_off, q_terms, 10)
    assert np.all(on["n"] == 10)
    _properties(on, 10, c.n_docs, "C4 pruned")
    sub = 2000
    sub_off, sub_terms = q_off[:sub + 1], q_terms[:q_off[sub]]
    ix.set_option("prune", 0)
    off = ix.search_batch(sub_off, sub_terms, 10)
    for key in ("doc", "score", "score64", "n"):
        assert np.array_equal(on[key][:sub], off[key]), f"C4: pruning changed `{key}`"
    assert on["stats"].postings_fetched < on["stats"].postings
    oix = oracle_index(orc, c)
    _sample_vs_oracle(on, oix, q_off, q_terms, 10, list(range(0, sub, 167)) + list(range(sub, 100_000, 9973)), "C4")
    ix.close()


def test_config5_25M_docs_mixed_queries(m, orc):
    """configs[4]: 25M docs (vocab 100k uniform, 128 terms/doc: 26 GB of postings, 39 GB of index in HBM), 1M
    mixed-length (1..8 term) queries, top-10 — one GPU's worth here; sharding across ranks is
    tests/test_sharding_gloo.py + bench.py --workload c5."""
    import psutil
    if psutil.virtual_memory().available < 110e9:
        pytest.skip("needs ~100 GB of host memory for the 25M-doc CSR + the oracle's copy")
    c = m.synth_corpus(0xB25C0DE5, 25_000_000, 100_000, 128)
    q_off, q_terms = m.synth_queries(0xB25C0DE5 + 1000, 1_000_000, 100_000, 1, 8, c.post_off)
    ix = m.Index.from_corpus(c)
    res = ix.search_batch(q_off, q_terms, 10)
    assert np.all(res["n"] == 10)
    _properties(res, 10, c.n_docs, "C5")
    oix = oracle_index(orc, c)
    _sample_vs_oracle(res, oix, q_off, q_terms, 10, range(0, 1_000_000, 15_873), "C5")              # 64 queries
    ix.close()
