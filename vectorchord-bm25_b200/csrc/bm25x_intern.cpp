// bm25x_intern.cpp — token interning (crates/bm25/src/vector.rs:19-35): the 16-byte key of a token.
//
//   short tokens (< 16 bytes, no NUL byte): the bytes themselves, zero padded;
//   everything else: the first 16 bytes of blake3::keyed_hash(seed, token), a zero last byte replaced by 1 so that a
//   hashed key can never collide with a padded short token.
//
// The reference takes BLAKE3 from the `blake3` crate (Cargo.lock: blake3 1.8.4), which is not vendored in
// the reference tree; the function below restates the published BLAKE3 algorithm (keyed_hash mode, full chunk tree) in
// portable C++.  Host code, one token per call; the tsvector casts intern whole batches on the GPU with the same
// algorithm (bm25x_tsvector.cu), and the tests hold the two to the same bits.
#include <stdint.h>
#include <string.h>

#include "../../include/bm25x.h"

namespace {

constexpr uint32_t IV[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au,
                            0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
constexpr uint8_t PERM[16] = {2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8};
enum : uint32_t { CHUNK_START = 1, CHUNK_END = 2, PARENT = 4, ROOT = 8, KEYED_HASH = 16 };
constexpr size_t BLOCK_LEN = 64, CHUNK_LEN = 1024;

inline uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
inline void g(uint32_t *s, int a, int b, int c, int d, uint32_t mx, uint32_t my) {
    s[a] = s[a] + s[b] + mx;
    s[d] = rotr(s[d] ^ s[a], 16);
    s[c] = s[c] + s[d];
    s[b] = rotr(s[b] ^ s[c], 12);
    s[a] = s[a] + s[b] + my;
    s[d] = rotr(s[d] ^ s[a], 8);
    s[c] = s[c] + s[d];
    s[b] = rotr(s[b] ^ s[c], 7);
}

// The compression function; out[0..8) = new chaining value (the first 8 words of the extended output).
void compress(const uint32_t cv[8], const uint32_t block[16], uint64_t counter, uint32_t block_len, uint32_t flags,
              uint32_t out[8]) {
    uint32_t s[16] = {cv[0], cv[1], cv[2], cv[3], cv[4], cv[5], cv[6], cv[7], IV[0], IV[1], IV[2], IV[3],
                      (uint32_t)counter, (uint32_t)(counter >> 32), block_len, flags};
    uint32_t m[16];
    memcpy(m, block, sizeof m);
    for (int r = 0; r < 7; r++) {
        g(s, 0, 4, 8, 12, m[0], m[1]);
        g(s, 1, 5, 9, 13, m[2], m[3]);
        g(s, 2, 6, 10, 14, m[4], m[5]);
        g(s, 3, 7, 11, 15, m[6], m[7]);
        g(s, 0, 5, 10, 15, m[8], m[9]);
        g(s, 1, 6, 11, 12, m[10], m[11]);
        g(s, 2, 7, 8, 13, m[12], m[13]);
        g(s, 3, 4, 9, 14, m[14], m[15]);
        uint32_t t[16];
        for (int i = 0; i < 16; i++) t[i] = m[PERM[i]];
        memcpy(m, t, sizeof m);
    }
    for (int i = 0; i < 8; i++) out[i] = s[i] ^ s[i + 8];
}

void load_block(const uint8_t *p, size_t n, uint32_t w[16]) {
    uint8_t buf[BLOCK_LEN] = {0};
    memcpy(buf, p, n);
    for (int i = 0; i < 16; i++)
        w[i] = (uint32_t)buf[4 * i] | (uint32_t)buf[4 * i + 1] << 8 | (uint32_t)buf[4 * i + 2] << 16 |
               (uint32_t)buf[4 * i + 3] << 24;
}

// A node whose compression has not been finalised yet (it may still turn out to be the root).
struct Output {
    uint32_t cv[8], block[16];
    uint64_t counter;
    uint32_t block_len, flags;
    void chaining_value(uint32_t out[8]) const { compress(cv, block, counter, block_len, flags, out); }
};

// One chunk (<= 1024 bytes, the last one possibly empty only for an empty input) → its last-block Output.
Output chunk_output(const uint32_t key[8], const uint8_t *p, size_t n, uint64_t chunk_index, uint32_t base_flags) {
    uint32_t cv[8];
    memcpy(cv, key, sizeof cv);
    size_t off = 0;
    uint32_t start = CHUNK_START;
    while (n - off > BLOCK_LEN) {
        uint32_t w[16];
        load_block(p + off, BLOCK_LEN, w);
        compress(cv, w, chunk_index, BLOCK_LEN, base_flags | start, cv);
        start = 0;
        off += BLOCK_LEN;
    }
    Output o;
    memcpy(o.cv, cv, sizeof cv);
    load_block(p + off, n - off, o.block);
    o.counter = chunk_index;
    o.block_len = (uint32_t)(n - off);
    o.flags = base_flags | start | CHUNK_END;
    return o;
}

Output parent_output(const uint32_t left[8], const uint32_t right[8], const uint32_t key[8], uint32_t base_flags) {
    Output o;
    memcpy(o.cv, key, sizeof o.cv);
    memcpy(o.block, left, 32);
    memcpy(o.block + 8, right, 32);
    o.counter = 0;
    o.block_len = BLOCK_LEN;
    o.flags = base_flags | PARENT;
    return o;
}

// First 16 bytes of BLAKE3 keyed_hash(key, data).
void blake3_keyed_16(const uint8_t key_bytes[32], const uint8_t *data, size_t len, uint8_t out[16]) {
    uint32_t key[8];
    for (int i = 0; i < 8; i++)
        key[i] = (uint32_t)key_bytes[4 * i] | (uint32_t)key_bytes[4 * i + 1] << 8 | (uint32_t)key_bytes[4 * i + 2] << 16 |
                 (uint32_t)key_bytes[4 * i + 3] << 24;
    uint32_t stack[54][8];  // chaining values of completed subtrees, one per set bit of the chunk count
    int depth = 0;
    uint64_t chunk = 0;
    size_t off = 0;
    while (len - off > CHUNK_LEN) {  // every chunk but the last: fold into the tree
        uint32_t cv[8];
        chunk_output(key, data + off, CHUNK_LEN, chunk, KEYED_HASH).chaining_value(cv);
        uint64_t total = chunk + 1;  // completed chunks so far: merge one subtree per trailing zero bit
        while ((total & 1) == 0) {
            uint32_t merged[8];
            parent_output(stack[depth - 1], cv, key, KEYED_HASH).chaining_value(merged);
            memcpy(cv, merged, sizeof cv);
            depth--;
            total >>= 1;
        }
        memcpy(stack[depth++], cv, sizeof cv);
        chunk++;
        off += CHUNK_LEN;
    }
    Output o = chunk_output(key, data + off, len - off, chunk, KEYED_HASH);
    while (depth > 0) {  // the right edge of the tree, bottom up
        uint32_t cv[8];
        o.chaining_value(cv);
        o = parent_output(stack[--depth], cv, key, KEYED_HASH);
    }
    uint32_t root[8];
    compress(o.cv, o.block, 0 /* root output block 0 */, o.block_len, o.flags | ROOT, root);
    // NB: for a root that is a chunk the counter field carries the output block index (0), not the chunk index —
    // a single-chunk input has chunk index 0 anyway; a parent has counter 0 by construction.
    for (int i = 0; i < 4; i++) {
        out[4 * i] = (uint8_t)root[i];
        out[4 * i + 1] = (uint8_t)(root[i] >> 8);
        out[4 * i + 2] = (uint8_t)(root[i] >> 16);
        out[4 * i + 3] = (uint8_t)(root[i] >> 24);
    }
}

}  // namespace

void bm25x_set_error(const char *fmt, ...);

extern "C" int bm25x_intern(const uint8_t seed[32], const uint8_t *token, size_t len, uint8_t key_out[BM25X_KEY_WIDTH]) {
    if (!seed || (!token && len) || !key_out) {
        bm25x_set_error("bm25x_intern: null argument");
        return BM25X_ERR_INVALID;
    }
    if (len < BM25X_KEY_WIDTH && (len == 0 || memchr(token, 0, len) == nullptr)) {  // vector.rs:21-24
        memset(key_out, 0, BM25X_KEY_WIDTH);
        if (len) memcpy(key_out, token, len);
        return BM25X_OK;
    }
    blake3_keyed_16(seed, token, len, key_out);  // vector.rs:26-29: first WIDTH bytes of the keyed hash
    if (key_out[BM25X_KEY_WIDTH - 1] == 0) key_out[BM25X_KEY_WIDTH - 1] = 1;  // vector.rs:30-32
    return BM25X_OK;
}

// Test hook: the raw 16-byte keyed-hash prefix without the interning rules (known-answer tests).
extern "C" int bm25x_blake3_keyed16(const uint8_t key[32], const uint8_t *data, size_t len, uint8_t out[16]) {
    if (!key || (!data && len) || !out) return BM25X_ERR_INVALID;
    blake3_keyed_16(key, data, len, out);
    return BM25X_OK;
}
