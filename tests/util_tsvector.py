"""PostgreSQL tsvectors as bm25x_tsvectors takes them, and the numpy restatement of the reference's casts over them
(src/datatype/tsvector.rs:84-127: vector::intern of every lexeme, sorted by key, equal keys merged with their position
counts summed with saturation) over the host bm25x.intern.

A batch is a dict(ent_off, entries, byte_off, data): vector i = its WordEntry words entries[ent_off[i]:ent_off[i+1]]
(bit 0 haspos, bits 1..11 len, bits 12..31 pos) and its lexeme area data[byte_off[i]:byte_off[i+1]]: each lexeme at pos,
and with haspos, at SHORTALIGN(pos + len), the u16 number of positions and the u16 WordEntryPos words."""
import numpy as np


def pack_ids(vec_lens, word_flat, word_off, wid, npos):
    """Vectors of vec_lens[i] entries each, entry j = word wid[j] (bytes word_flat[word_off[w]:word_off[w+1]]) with
    npos[j] positions 1..npos[j] (-1: no positions), in the order given (duplicates and any order allowed: the casts sort
    and merge)."""
    vec_lens = np.asarray(vec_lens, np.int64)
    word_off = np.asarray(word_off, np.int64)
    wid = np.asarray(wid, np.int64)
    npos = np.asarray(npos, np.int64)
    lens = word_off[wid + 1] - word_off[wid]
    has = npos >= 0
    cnt = np.maximum(npos, 0)
    # bytes of each entry in its area: the lexeme, then (haspos) pad to even, u16 count, u16 positions
    size = np.where(has, ((lens + 1) & ~1) + 2 + 2 * cnt, lens)
    ent_off = np.zeros(len(vec_lens) + 1, np.uint64)
    ent_off[1:] = np.cumsum(vec_lens)
    vec = np.repeat(np.arange(len(vec_lens)), vec_lens)
    starts = np.cumsum(size) - size                              # global offset of each entry's bytes
    per_vec = np.bincount(vec, weights=size, minlength=len(vec_lens)).astype(np.int64)
    byte_off = np.zeros(len(vec_lens) + 1, np.uint64)
    byte_off[1:] = np.cumsum(per_vec)
    pos = starts - byte_off[:-1].astype(np.int64)[vec]
    assert (pos < (1 << 20)).all() and (lens < (1 << 11)).all()
    entries = ((pos << 12) | (lens << 1) | has.astype(np.int64)).astype(np.uint32)
    data = np.zeros(int(byte_off[-1]), np.uint8)
    total = int(lens.sum())
    if total:
        k = np.arange(total) - np.repeat(np.cumsum(lens) - lens, lens)   # byte index inside its lexeme
        data[np.repeat(starts, lens) + k] = np.asarray(word_flat, np.uint8)[np.repeat(word_off[wid], lens) + k]
    h = np.nonzero(has)[0]
    if len(h):
        at = starts[h] + ((lens[h] + 1) & ~1)
        data[at] = cnt[h] & 0xFF
        data[at + 1] = cnt[h] >> 8
        # positions 1..npos as WordEntryPos (weight 0): u16 little-endian after the count
        reps = cnt[h]
        base = np.repeat(at + 2, reps)
        k = np.arange(int(reps.sum())) - np.repeat(np.cumsum(reps) - reps, reps)
        p = (k + 1) & 0x3FFF
        data[base + 2 * k] = p & 0xFF
        data[base + 2 * k + 1] = p >> 8
    return dict(ent_off=ent_off, entries=entries, byte_off=byte_off, data=data)


def assemble(vectors):
    """A batch from (area u8, entries u32) per vector: the WordEntry words as given, each vector's lexeme area as given
    (it may hold bytes no entry points at)."""
    lens = [len(e) for _, e in vectors]
    sizes = [len(a) for a, _ in vectors]
    ent_off = np.zeros(len(vectors) + 1, np.uint64)
    ent_off[1:] = np.cumsum(lens)
    byte_off = np.zeros(len(vectors) + 1, np.uint64)
    byte_off[1:] = np.cumsum(sizes)
    entries = np.concatenate([np.asarray(e, np.uint32) for _, e in vectors]) if vectors else np.zeros(0, np.uint32)
    data = np.concatenate([np.asarray(a, np.uint8) for a, _ in vectors]) if vectors else np.zeros(0, np.uint8)
    return dict(ent_off=ent_off, entries=entries, byte_off=byte_off, data=data)


def word_table(words):
    """A list of bytes as (flat u8, offsets [len + 1])."""
    off = np.zeros(len(words) + 1, np.int64)
    off[1:] = np.cumsum([len(w) for w in words])
    return np.frombuffer(b"".join(words), np.uint8).copy(), off


def pack(vec_lens, lexemes, npos):
    """pack_ids over a list of lexemes (bytes), entry j = lexemes[j], npos[j] positions or None."""
    flat, off = word_table(lexemes)
    return pack_ids(vec_lens, flat, off, np.arange(len(lexemes)), [-1 if p is None else p for p in npos])


def write_tsvectors(vectors):
    """vectors: per vector a list of (lexeme bytes, positions list or None), written in that order; PostgreSQL keeps
    entries sorted and distinct, which pack_sorted gives."""
    lens = [len(v) for v in vectors]
    lex = [x for v in vectors for x, _ in v]
    npos = [None if p is None else len(p) for v in vectors for _, p in v]
    return pack(lens, lex, npos)


def pack_sorted(docs):
    """PostgreSQL's layout of {lexeme: positions} per vector: entries sorted by lexeme (tsCompareString), distinct."""
    return write_tsvectors([sorted(d.items()) for d in docs])


def decode(tsv):
    """Per entry: (vector, len, pos, haspos, count) as numpy arrays (TsVectorBorrowed::iter)."""
    ent_off = np.asarray(tsv["ent_off"], np.int64)
    e = np.asarray(tsv["entries"], np.uint32).astype(np.int64)
    vec = np.repeat(np.arange(len(ent_off) - 1), np.diff(ent_off))
    has, length, pos = e & 1, (e >> 1) & 0x7FF, e >> 12
    data = np.asarray(tsv["data"], np.uint8)
    area = np.asarray(tsv["byte_off"], np.int64)[:-1][vec] if len(vec) else np.zeros(0, np.int64)
    at = area + ((pos + length + 1) & ~1)
    count = np.zeros(len(e), np.int64)
    hh = np.nonzero(has)[0]
    count[hh] = data[at[hh]].astype(np.int64) | (data[at[hh] + 1].astype(np.int64) << 8)
    return vec, length, area + pos, has.astype(bool), count


def entry_keys(intern, seed, tsv):
    """vector::intern of every entry's lexeme ([E, 16] u8): short lexemes without NUL zero-padded in numpy, the others
    through the host bm25x_intern (once per distinct lexeme)."""
    vec, length, start, _, _ = decode(tsv)
    data = np.asarray(tsv["data"], np.uint8)
    E = len(length)
    keys = np.zeros((E, 16), np.uint8)
    j = np.arange(16)
    short = length < 16
    if E:
        mask = j[None, :] < length[:, None]
        idx = np.where(mask, start[:, None] + j[None, :], 0)
        got = np.where(mask, data[np.minimum(idx, max(len(data) - 1, 0))] if len(data) else 0, 0).astype(np.uint8)
        nul = (mask & (got == 0)).any(axis=1)
        copy = short & ~nul
        keys[copy] = got[copy]
        cache = {}
        for i in np.nonzero(~copy)[0]:
            lex = bytes(data[start[i]:start[i] + length[i]])
            if lex not in cache:
                cache[lex] = np.frombuffer(intern(seed, lex), np.uint8)
            keys[i] = cache[lex]
    return keys


def cast(intern, seed, tsv, as_query=False, keys=None):
    """The restated cast_tsvector_to_document / cast_tsvector_to_query: (off u64 [n+1], keys [E', 16], tf u32 [E'] or
    None).  keys: the entries' keys when already computed."""
    vec, _, _, _, count = decode(tsv)
    n = len(tsv["ent_off"]) - 1
    k = entry_keys(intern, seed, tsv) if keys is None else keys
    w = k.view(">u8").reshape(-1, 2) if len(k) else np.zeros((0, 2), np.uint64)
    order = np.lexsort((w[:, 1], w[:, 0], vec))
    v, ks, c = vec[order], k[order], count[order]
    ws = w[order]
    first = np.ones(len(order), bool)
    if len(order):
        first[1:] = (v[1:] != v[:-1]) | (ws[1:, 0] != ws[:-1, 0]) | (ws[1:, 1] != ws[:-1, 1])
    heads = np.nonzero(first)[0]
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(v[heads], minlength=n)) if len(heads) else 0
    tf = None
    if not as_query:
        sums = np.add.reduceat(c, heads) if len(heads) else np.zeros(0, np.int64)
        tf = np.minimum(sums, 0xFFFFFFFF).astype(np.uint32)            # Saturating<u32>
    return off, ks[heads], tf


CHUNK_ENT, CHUNK_BYTES, CHUNK_VEC = 1 << 22, 1 << 26, 1 << 22   # the cast's chunk limits (bm25x_tsvector.cu)


def cast_cuts(tsv):
    """The restated cut loop of run_cast: per chunk (a, b, rule, ne), vectors [a, b) holding ne entries, closed by
    "end" (the batch), "vectors" (CHUNK_VEC of them), "single" (vector a alone exceeds a limit), "entries" or "bytes"
    (vector b would take the chunk past CHUNK_ENT entries or CHUNK_BYTES lexeme-area bytes).  A chunk with ne == 0 is
    skipped by the cast."""
    ent = np.asarray(tsv["ent_off"], np.int64)
    byt = np.asarray(tsv["byte_off"], np.int64)
    n = len(ent) - 1
    out, a = [], 0
    while a < n:
        # b = a + 1 + the vectors after a that fit: a prefix of a monotone test, found by binary search
        stop = min(n, a + CHUNK_VEC)
        b = a + 1
        if b < stop:
            lo = np.searchsorted(ent[b + 1:stop + 1], ent[a] + CHUNK_ENT, side="right")
            hi = np.searchsorted(byt[b + 1:stop + 1], byt[a] + CHUNK_BYTES, side="right")
            b += int(min(lo, hi))
        if b == n:
            rule = "end"
        elif b - a == CHUNK_VEC:
            rule = "vectors"
        elif b == a + 1 and (ent[b] - ent[a] > CHUNK_ENT or byt[b] - byt[a] > CHUNK_BYTES):
            rule = "single"
        elif ent[b + 1] - ent[a] > CHUNK_ENT:
            rule = "entries"
        else:
            rule = "bytes"
        out.append((a, b, rule, int(ent[b] - ent[a])))
        a = b
    return out


def byte_cut_batch(seed=21):
    """Cut by bytes: areas of about 1 MiB (a few long lexemes, 1 000..2 047 bytes, at the front; the rest padding no entry
    points into).  Chunk 0's 64 areas end exactly at CHUNK_BYTES; chunk 1's 64th vector would end one byte past it.
    Returns (tsv, words, word id per entry)."""
    rng = np.random.default_rng(seed)
    words = list(dict.fromkeys(bytes(rng.integers(97, 123, int(rng.integers(1000, 2048)), dtype=np.uint8))
                               for _ in range(300)))
    M = 1 << 20
    sizes = [M] * 64 + [M + 1] + [M] * 62 + [M] + [20_000, 0, 300_000, 0, 30_000]
    vectors, wid_all = [], []
    for v, size in enumerate(sizes):
        if size == 0:
            vectors.append((np.zeros(size, np.uint8), np.zeros(0, np.uint32)))
            continue
        k = int(rng.integers(1, 5 if size < M else 12))
        wids = rng.choice(len(words), size=k, replace=False)
        area, at = bytearray(), []
        for w in wids:
            at.append(len(area))
            x = words[w]
            area += x + (b"\0" if len(x) % 2 else b"") + int(rng.integers(1, 9)).to_bytes(2, "little")
        assert len(area) <= size
        area += bytes(size - len(area))
        pick = rng.integers(0, k, int(rng.integers(20, 200)))
        ents = np.array([(at[p] << 12) | (len(words[wids[p]]) << 1) | 1 for p in pick], np.uint32)
        vectors.append((np.frombuffer(bytes(area), np.uint8), ents))
        wid_all.append(wids[pick])
    return assemble(vectors), words, np.concatenate(wid_all)


def synthetic(rng, n, len_min, len_max, vocab, long_frac, max_pos=4, long_min=16, long_max=64):
    """n tsvectors of about len_min..len_max distinct lexemes drawn (Zipf-like) from a vocabulary of `vocab` distinct
    lowercase words, long_frac of them long_min..long_max bytes (the hash path), the rest 1..15 (the copy path), each with
    1..max_pos positions; entries sorted by word id.  Returns (tsv, words, word id per entry)."""
    n_long = int(round(vocab * long_frac))
    wl = np.concatenate([rng.integers(long_min, long_max + 1, n_long), rng.integers(1, 16, vocab - n_long)])
    rng.shuffle(wl)
    raw = rng.integers(97, 123, int(wl.sum()), dtype=np.uint8).tobytes()
    cut = np.concatenate([[0], np.cumsum(wl)])
    words = list(dict.fromkeys(raw[cut[i]:cut[i + 1]] for i in range(vocab)))
    V = len(words)
    p = 1.0 / np.arange(1, V + 1) ** 0.8
    p /= p.sum()
    want = rng.integers(len_min, len_max + 1, n)
    vec = np.repeat(np.arange(n), want)
    wid = rng.choice(V, size=len(vec), p=p)
    pair = np.unique(vec.astype(np.int64) * V + wid)                # distinct per vector, as PostgreSQL keeps them
    vec, wid = pair // V, pair % V
    lens = np.bincount(vec, minlength=n)
    npos = rng.integers(1, max_pos + 1, len(wid))
    flat, off = word_table(words)
    return pack_ids(lens, flat, off, wid, npos), words, wid
