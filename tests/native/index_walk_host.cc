// CPU check of K2's word-window Index.db reader (index_walk.cuh: IdxCursor, iw_entry), meant to be built with -fsanitize=address,undefined.
// Test infrastructure only.
// Usage: index_walk_host <iterations> [<Index.db path> <Data.db length>]...
// Every Index.db image lives in a heap buffer that holds `align` bytes before it (the cursor's aligned loads may start there, as they do in
// K2's workspace) and ends exactly IW_PAD bytes past its last byte. On it:
//   - the cursor's parse equals a byte-wise parse with idx_entry's checks (compact.cu) entry for entry, walking the whole file and walking
//     from every 128th entry (one Summary interval per cursor, as k_index_walk_count / _emit do), with key prefix and token;
//   - truncated and damaged images stop both parses at the same offset, and both agree at arbitrary (non-entry) offsets;
// and the window's Murmur3 equals the oracle's murmur3_token for random keys of length 0..80 at every alignment.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <random>
#include <string>
#include "../../cassandra_b200/csrc/index_walk.cuh"
#include "../../oracle/codec.h"

using namespace b200c;

// ---- the byte-wise reference: idx_entry (compact.cu) and vint_read (common.cuh) on plain bytes ---------------------------------------
static int ref_vint(const uint8_t* p, const uint8_t* end, uint64_t* v) {
    if (p >= end) return 0;
    const uint32_t first = p[0];
    if (first < 0x80) { *v = first; return 1; }
    int extra = 0; for (uint32_t x = first; x & 0x80; x = (x << 1) & 0xFF) extra++;
    if (p + 1 + extra > end) return 0;
    uint64_t r = extra == 8 ? 0 : (first & (0xFFu >> extra));
    for (int i = 0; i < extra; i++) r = (r << 8) | p[1 + i];
    *v = r;
    return 1 + extra;
}
struct Ref { uint64_t len, pos; uint32_t kl; uint64_t pre; int64_t tok; };
static Ref ref_entry(const uint8_t* b, uint64_t ilen, uint64_t ulen, uint64_t o, bool murmur) {
    Ref r{0, 0, 0, 0, 0};
    if (o + 2 > ilen) return r;
    const uint32_t kl = ((uint32_t)b[o] << 8) | b[o + 1];
    uint64_t p = o + 2 + kl;
    if (p + 2 > ilen) return r;
    uint64_t pos, ps;
    int n = ref_vint(b + p, b + ilen, &pos); if (!n) return r; p += n;
    n = ref_vint(b + p, b + ilen, &ps); if (!n) return r; p += n;
    if (ps > 0x7FFFFFFFull || p + ps > ilen) return r;
    if (pos >= ulen || pos + 2 + kl + 2 > ulen) return r;
    const uint8_t* key = b + o + 2;
    uint64_t pre = 0; for (uint32_t q = 0; q < 8; q++) pre = (pre << 8) | (q < kl ? key[q] : 0);      // order_token_of / k_index_emit
    r.len = p + ps - o; r.pos = pos; r.kl = kl; r.pre = pre;
    r.tok = murmur ? oracle::murmur3_token(key, kl) : (int64_t)(pre ^ 0x8000000000000000ull);
    return r;
}

static int failures = 0;
#define CHECK(cond, ...) do { if (!(cond)) { if (failures++ < 20) { fprintf(stderr, __VA_ARGS__); fputc('\n', stderr); } } } while (0)

// an image in a buffer that ends exactly IW_PAD bytes past it, `align` bytes after a 16-byte boundary
struct Img {
    uint8_t* alloc; const uint8_t* p; uint64_t len;
    Img(const uint8_t* src, uint64_t n, int align) : len(n) {
        if (posix_memalign((void**)&alloc, 16, align + n + IW_PAD)) abort();
        memset(alloc, 0xC3, align + n + IW_PAD);
        if (n) memcpy(alloc + align, src, n);
        p = alloc + align;
    }
    ~Img() { free(alloc); }
};

static bool same(const Ref& r, uint64_t len, const IdxEntry& e, bool key) {
    if (r.len != len) return false;
    if (!len) return true;
    return r.pos == e.pos && r.kl == e.kl && (!key || (r.pre == e.pre && r.tok == e.tok));
}

// walks both parsers from `from` until one stops (or `stop`); returns the offset where they stopped, ~0 on a mismatch
static uint64_t walk(const Img& m, uint64_t ulen, uint64_t from, uint64_t stop, bool key, bool murmur, std::vector<uint64_t>* starts, const char* what) {
    IdxCursor c; c.init(m.p, m.len);
    uint64_t o = from;
    while (o < stop) {
        const Ref r = ref_entry(m.p, m.len, ulen, o, murmur);
        IdxEntry e{0, 0, 0, 0};
        const uint64_t len = key ? iw_entry<true>(c, o, ulen, murmur, e) : iw_entry<false>(c, o, ulen, murmur, e);
        if (!same(r, len, e, key)) { CHECK(false, "%s: entry at %llu differs (len %llu vs %llu, pos %llu vs %llu, kl %u vs %u, tok %lld vs %lld)", what,
                                           (unsigned long long)o, (unsigned long long)r.len, (unsigned long long)len, (unsigned long long)r.pos, (unsigned long long)e.pos,
                                           r.kl, e.kl, (long long)r.tok, (long long)e.tok); return ~0ull; }
        if (!len) return o;
        if (starts) starts->push_back(o);
        o += len;
    }
    return o;
}

static void check_file(const std::vector<uint8_t>& f, uint64_t ulen, std::mt19937_64& rng, const std::string& name) {
    std::vector<uint64_t> starts;
    for (int align = 0; align < 16; align += 5) {
        Img m(f.data(), f.size(), align);
        for (int mm = 0; mm < 2; mm++) {
            std::vector<uint64_t>* st = (align == 0 && mm == 0) ? &starts : nullptr;
            const uint64_t end = walk(m, ulen, 0, m.len, true, mm == 0, st, name.c_str());
            CHECK(end == m.len, "%s: the walk stopped at %llu of %llu", name.c_str(), (unsigned long long)end, (unsigned long long)m.len);
        }
        // one cursor per Summary interval (every 128th entry), count walk and emit walk; the emit walk parses the next interval's first entry too
        for (size_t s = 0; s < starts.size(); s += 128) {
            const uint64_t from = starts[s], to = s + 128 < starts.size() ? starts[s + 128] : m.len;
            CHECK(walk(m, ulen, from, to, false, true, nullptr, name.c_str()) == to, "%s: interval at %llu did not land", name.c_str(), (unsigned long long)from);
            IdxCursor c; c.init(m.p, m.len); IdxEntry e{0, 0, 0, 0};
            uint64_t o = from;
            while (o < to) { const uint64_t l = iw_entry<true>(c, o, ulen, true, e); if (!l) break; o += l; }
            if (to < m.len) { const uint64_t l = iw_entry<true>(c, to, ulen, true, e); CHECK(same(ref_entry(m.p, m.len, ulen, to, true), l, e, true), "%s: next interval's first entry", name.c_str()); }
        }
        // arbitrary offsets (most are not entry starts): both parsers must agree on every one
        for (int k = 0; k < 2000 && m.len; k++) {
            const uint64_t o = rng() % (m.len + 4);
            IdxCursor c; c.init(m.p, m.len); IdxEntry e{0, 0, 0, 0};
            const uint64_t l = iw_entry<true>(c, o, ulen, true, e);
            CHECK(same(ref_entry(m.p, m.len, ulen, o, true), l, e, true), "%s: offset %llu", name.c_str(), (unsigned long long)o);
        }
    }
    // truncated images (the buffer ends IW_PAD bytes past the cut) and damaged ones: both parsers stop at the same offset
    for (int k = 0; k < 40 && !f.empty(); k++) {
        const uint64_t cut = k < 8 && !starts.empty() ? starts[rng() % starts.size()] + 1 + rng() % 20 : rng() % (f.size() + 1);
        const uint64_t n = cut < f.size() ? cut : f.size();
        Img m(f.data(), n, (int)(rng() % 16));
        walk(m, ulen, 0, m.len, true, true, nullptr, (name + " truncated").c_str());
        std::vector<uint8_t> d = f;
        for (int q = 0; q < 1 + (int)(rng() % 4); q++) { const uint64_t x = rng() % d.size(); d[x] = (uint8_t)(rng() % 3 == 0 ? 0xFF : rng()); }
        Img m2(d.data(), d.size(), (int)(rng() % 16));
        walk(m2, ulen, 0, m2.len, true, true, nullptr, (name + " damaged").c_str());
        walk(m2, ulen / 2, 0, m2.len, false, true, nullptr, (name + " short Data.db").c_str());
    }
    printf("  %s: %zu entries, %zu bytes\n", name.c_str(), starts.size(), f.size());
}

// synthetic entries with every vint width and key length 0..80, promoted-index payloads included
static std::vector<uint8_t> random_index(std::mt19937_64& rng, uint64_t* ulen) {
    std::vector<uint8_t> f;
    uint64_t pos = 0;
    const int n = 1 + (int)(rng() % 600);
    auto vint = [&](uint64_t v) {                          // VIntCoding.writeUnsignedVInt
        const int extra = ((639 - __builtin_clzll(v | 1) * 9) >> 6) - 1;
        if (extra == 0) { f.push_back((uint8_t)v); return; }
        f.push_back(extra == 8 ? 0xFF : (uint8_t)(((0xFF00u >> extra) & 0xFF) | (uint32_t)(v >> (8 * extra))));
        for (int i = extra - 1; i >= 0; i--) f.push_back((uint8_t)(v >> (8 * i)));
    };
    for (int k = 0; k < n; k++) {
        const uint32_t kl = rng() % 5 == 0 ? (uint32_t)(rng() % 81) : 8;
        f.push_back((uint8_t)(kl >> 8)); f.push_back((uint8_t)kl);
        for (uint32_t q = 0; q < kl; q++) f.push_back((uint8_t)rng());
        vint(pos);
        const uint32_t ps = rng() % 7 == 0 ? (uint32_t)(rng() % 300) : 0;
        vint(ps);
        for (uint32_t q = 0; q < ps; q++) f.push_back((uint8_t)rng());
        pos += 2 + kl + 2 + (rng() % 3 == 0 ? rng() % (1ull << (7 * (1 + rng() % 6))) : rng() % 200);
    }
    *ulen = pos + 1;
    return f;
}

int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 200;
    std::mt19937_64 rng(0x1D3A11C);
    for (int a = 2; a + 1 < argc; a += 2) {
        FILE* fp = fopen(argv[a], "rb"); if (!fp) { fprintf(stderr, "cannot open %s\n", argv[a]); return 2; }
        std::vector<uint8_t> f; uint8_t buf[65536]; size_t n;
        while ((n = fread(buf, 1, sizeof(buf), fp)) > 0) f.insert(f.end(), buf, buf + n);
        fclose(fp);
        check_file(f, strtoull(argv[a + 1], nullptr, 10), rng, argv[a]);
    }
    for (int it = 0; it < iters; it++) { uint64_t ulen; const std::vector<uint8_t> f = random_index(rng, &ulen); check_file(f, ulen, rng, "random " + std::to_string(it)); }
    // Murmur3 from the window against the oracle: every length 0..80 at every alignment, inside a buffer that ends IW_PAD bytes past the key
    long keys = 0;
    for (int len = 0; len <= 80; len++)
        for (int align = 0; align < 16; align++)
            for (int rep = 0; rep < 4; rep++) {
                std::vector<uint8_t> k(len);
                for (auto& b : k) b = (uint8_t)(rep == 0 ? 0x80 | rng() : rep == 1 ? rng() & 0x7F : rng());
                Img m(k.data(), k.size(), align);
                IdxCursor c; c.init(m.p, m.len);
                CHECK(c.murmur3(0, (uint32_t)len) == oracle::murmur3_token(k.data(), k.size()), "murmur3 of %d bytes at alignment %d", len, align);
                keys++;
            }
    if (failures) { fprintf(stderr, "%d failures\n", failures); return 1; }
    printf("index_walk_host ok: %d files + %d random indexes, %ld keys hashed\n", (argc - 2) / 2, iters, keys);
    return 0;
}
