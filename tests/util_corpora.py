"""Corpora that more than one test module searches: the synthetic shapes of the parity and stored-block tests, the
33..64-term shapes, posting lists given term by term, the adversarial sharded corpus and its shard bounds, and the
sqllogictest passages of the reference's goldens."""
import numpy as np

# synth_corpus / synth_queries arguments of the parity shapes
PARITY_CONFIGS = [
    dict(name="C1", seed=0xB25C0DE1, n=1000, vocab=1000, lmin=32, lmax=32, zipf=0.0, nq=100, tmin=3, tmax=3),
    dict(name="varlen", seed=21, n=20000, vocab=3000, lmin=1, lmax=300, zipf=0.0, nq=80, tmin=1, tmax=8),
    dict(name="zipf", seed=22, n=30000, vocab=5000, lmin=16, lmax=96, zipf=1.0, nq=80, tmin=1, tmax=8),
    dict(name="dense", seed=23, n=5000, vocab=40, lmin=5, lmax=400, zipf=1.1, nq=60, tmin=1, tmax=8),
    dict(name="manyterms", seed=24, n=8000, vocab=600, lmin=8, lmax=64, zipf=0.8, nq=40, tmin=9, tmax=32),
    dict(name="ties", seed=25, n=50000, vocab=200, lmin=16, lmax=16, zipf=0.0, nq=60, tmin=1, tmax=4),
]

# synth_corpus arguments of the stored-block shapes
BLOCK_CONFIGS = [
    dict(name="C1", seed=0xB25C0DE1, n=1000, vocab=1000, lmin=32, lmax=32, zipf=0.0),      # only short (byte-packed) blocks
    dict(name="zipf", seed=22, n=30000, vocab=5000, lmin=16, lmax=96, zipf=1.0),           # full + short blocks, wide bit widths
    dict(name="dense", seed=23, n=5000, vocab=40, lmin=5, lmax=400, zipf=1.1),             # 1-2 bit deltas, large tf
    dict(name="ties", seed=25, n=50000, vocab=200, lmin=16, lmax=16, zipf=0.0),
]

TWO_PASS = [
    # uniform vocabulary: df is not monotone in the term id, so the two groups interleave in id order
    dict(name="uniform", seed=101, n=20000, vocab=1500, lmin=8, lmax=120, zipf=0.0, weighted=False),
    # dense: 72 terms, long documents (dense windows in pass 0)
    dict(name="dense", seed=102, n=4000, vocab=72, lmin=60, lmax=400, zipf=0.5, weighted=False),
    # Zipf, terms drawn by df: head terms pruned while group 1 is probed
    dict(name="zipf", seed=103, n=30000, vocab=3000, lmin=16, lmax=96, zipf=1.0, weighted=True),
]


def csr_corpus(rng, n_docs, lists, extra_len=0):
    """Term-major CSR from explicit posting lists [(doc ids, tfs)]; a document's length is its Σ tf plus up to
    `extra_len` tokens of terms outside the corpus (varied norms)."""
    off = np.zeros(len(lists) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d, _ in lists])
    post_doc = np.concatenate([np.asarray(d, np.uint32) for d, _ in lists])
    post_tf = np.concatenate([np.asarray(t, np.uint32) for _, t in lists])
    doc_len = np.bincount(post_doc, weights=post_tf, minlength=n_docs).astype(np.uint32)
    if extra_len:
        doc_len += rng.integers(0, extra_len + 1, size=n_docs).astype(np.uint32)
    return doc_len, off, post_doc, post_tf


def corpus_dict(n_docs, lists, doc_len=None):
    """The Index / ShardedIndex arguments of explicit posting lists [(doc ids, tfs)]; lengths Σ tf + 1 unless given."""
    off = np.zeros(len(lists) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d, _ in lists])
    post_doc = np.concatenate([np.asarray(d, np.uint32) for d, _ in lists])
    post_tf = np.concatenate([np.asarray(t, np.uint32) for _, t in lists])
    if doc_len is None:
        doc_len = np.bincount(post_doc, weights=post_tf, minlength=n_docs).astype(np.uint32) + 1
    return dict(n_docs=n_docs, doc_len=doc_len, n_terms=len(lists), post_off=off, post_doc=post_doc, post_tf=post_tf)


ADVERSARIAL_BOUNDS = [0, 997, 2001, 2002, 2003, 2301, 2600, 3333, 4000]


def adversarial_corpus():
    """The corpus of test_gpu_sharded.py::test_adversarial_bounds, and its random generator for what the test draws
    next."""
    rng = np.random.default_rng(3)
    N = 4000
    lists = []
    for t in range(60):                                   # ordinary terms over [0, 2000) and [2600, 4000)
        docs = np.sort(rng.choice(np.r_[0:2000, 2600:4000], size=int(rng.integers(5, 600)), replace=False))
        lists.append((docs, rng.integers(1, 6, size=len(docs))))
    lists.append((np.arange(2100, 2300), rng.integers(1, 4, size=200)))     # term 60: all postings in [2003, 2301)
    lists.append((np.array([2001]), np.array([3])))                          # term 61: one document, shard [2001, 2002)
    # [2301, 2600) holds no posting at all; [2002, 2003) has no query term
    return corpus_dict(N, lists, doc_len=rng.integers(1, 200, size=N).astype(np.uint32)), rng


# index options of the sharded kernel-path runs, on top of the defaults
SHARDED_PATHS = dict(default={}, seed_off={"seed": 0},
                     seeded_forced={"seed_dense_div": 0, "seed_prune_min": 0xFFFFFFFF},
                     twophase={"seed": 0, "twophase": 1}, prune_off={"prune": 0})


def slt_corpus(orc, golden, ids):
    """Corpus of the slt passages with 1-based ids in `ids`; lexeme id = rank of the lexeme string
    (reference keys are the raw bytes, vector.rs:19-35, compared bytewise)."""
    docs = [golden["doc_lexemes"][i - 1] for i in ids]
    vocab = sorted({w for d in docs for w in d})
    tid = {w: i for i, w in enumerate(vocab)}
    dd = []
    for d in docs:
        m = {}
        for w in d:
            m[tid[w]] = m.get(tid[w], 0) + 1
        dd.append(m)
    c = orc.Corpus.from_docs(dd, n_terms=len(vocab))
    assert list(c.doc_len) == [golden["doc_lengths"][i - 1] for i in ids]
    return c, tid
