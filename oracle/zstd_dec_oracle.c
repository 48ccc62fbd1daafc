/* zstd_dec_oracle.c -- plain-C restatement of the Zstandard decoder (RFC 8878).
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline
 * leg may load this.  It is the checker for the CUDA decoder (bit-exact output) and the
 * second, independent verifier of frames the CUDA encoder emits (the first being the
 * reference itself, oracle/_ref/libref_zstd.so).
 *
 * Parity pin: tests/test_oracle_zstd.py checks this file against
 *   - the reference's golden vector tests/regr-arc/test.txt.zstd (committed as a fixture), and
 *   - frames produced by the reference encoder (oracle/_ref) at levels -5..19, with/without
 *     checksum, multi-frame and skippable-frame concatenations.
 *
 * Reference functions restated (under /root/reference/C/zstd/):
 *   frame header / block loop ........ zstd_decompress.c:702 (ZSTD_decodeFrameHeader), :1275
 *   block header ..................... zstd_decompress_block.c:63-77 (ZSTD_getcBlockSize)
 *   literals section ................. zstd_decompress_block.c:134-340 (ZSTD_decodeLiteralsBlock)
 *   Huffman table read ............... entropy_common.c:242-305 (HUF_readStats), huf_decompress.c:385
 *   Huffman 1X/4X stream decode ...... huf_decompress.c:897,840
 *   FSE NCount read .................. entropy_common.c:42-188 (FSE_readNCount)
 *   FSE decode-table build ........... zstd_decompress_block.c:485-600 (ZSTD_buildFSETable_body)
 *   sequence header .................. zstd_decompress_block.c:695-775 (ZSTD_decodeSeqHeaders)
 *   sequence decode + repcodes ....... zstd_decompress_block.c:1229-1345 (ZSTD_decodeSequence)
 *   sequence execution ............... zstd_decompress_block.c:1001 (ZSTD_execSequence)
 *   skippable frames ................. zstd_decompress.c:482-489,587-600
 *   XXH64 content checksum ........... ../hashes/xxhash.c (XXH64), zstd_decompress.c (checksum check)
 */
#include <string.h>
#include <stdlib.h>
#include "zstd_format.h"
#include "oracle.h"

/* ---------------------------------------------------------------- XXH64 (seed 0) */
#define XP1 0x9E3779B185EBCA87ull
#define XP2 0xC2B2AE3D27D4EB4Full
#define XP3 0x165667B19E3779F9ull
#define XP4 0x85EBCA77C2B2AE63ull
#define XP5 0x27D4EB2F165667C5ull
static inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static inline uint64_t rd64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static inline uint64_t xround(uint64_t acc, uint64_t in) { return rotl64(acc + in * XP2, 31) * XP1; }
static inline uint64_t xmerge(uint64_t h, uint64_t v) { return (h ^ xround(0, v)) * XP1 + XP4; }
uint64_t b2zo_xxh64(const void *data, size_t len, uint64_t seed) {
    const uint8_t *p = (const uint8_t *)data, *end = p + len;
    uint64_t h;
    if (len >= 32) {
        uint64_t v1 = seed + XP1 + XP2, v2 = seed + XP2, v3 = seed, v4 = seed - XP1;
        do { v1 = xround(v1, rd64(p)); v2 = xround(v2, rd64(p + 8)); v3 = xround(v3, rd64(p + 16)); v4 = xround(v4, rd64(p + 24)); p += 32; }
        while (p + 32 <= end);
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = xmerge(h, v1); h = xmerge(h, v2); h = xmerge(h, v3); h = xmerge(h, v4);
    } else h = seed + XP5;
    h += (uint64_t)len;
    while (p + 8 <= end) { h ^= xround(0, rd64(p)); h = rotl64(h, 27) * XP1 + XP4; p += 8; }
    if (p + 4 <= end) { h ^= (uint64_t)rd32(p) * XP1; h = rotl64(h, 23) * XP2 + XP3; p += 4; }
    while (p < end) { h ^= (*p++) * XP5; h = rotl64(h, 11) * XP1; }
    h ^= h >> 33; h *= XP2; h ^= h >> 29; h *= XP3; h ^= h >> 32;
    return h;
}

/* ---------------------------------------------------------------- bit readers */
/* forward LSB-first reader (FSE NCount headers) */
typedef struct { const uint8_t *p; size_t size; size_t bitpos; } fwd_t;
static uint32_t fwd_peek(const fwd_t *b, int n) {     /* n <= 24; bytes past the end read as 0 */
    uint64_t v = 0; size_t byte = b->bitpos >> 3;
    for (int i = 0; i < 5; i++) if (byte + (size_t)i < b->size) v |= (uint64_t)b->p[byte + (size_t)i] << (8 * i);
    return (uint32_t)((v >> (b->bitpos & 7)) & ((1u << n) - 1));
}

/* backward reader: the last byte holds a 1-bit end mark above the data bits */
typedef struct { const uint8_t *p; int64_t bitpos; int overflow; } bwd_t;
static int bwd_init(bwd_t *b, const uint8_t *p, size_t size) {
    if (size == 0 || p[size - 1] == 0) return -1;
    b->p = p; b->overflow = 0;
    b->bitpos = (int64_t)(size - 1) * 8 + (int64_t)zf_highbit32(p[size - 1]);
    return 0;
}
/* read n bits (n <= 32); bits before the start of the buffer read as zero and set overflow */
static uint32_t bwd_read(bwd_t *b, int n) {
    if (n == 0) return 0;
    int64_t lo = b->bitpos - n;
    uint64_t v = 0;
    if (lo < 0) {
        b->overflow = 1;
        int avail = (int)b->bitpos;                       /* may be <= 0 */
        if (avail > 0) {
            uint64_t w = 0;
            for (int i = 0; i < 8 && i * 8 < avail; i++) w |= (uint64_t)b->p[i] << (8 * i);
            w &= (avail >= 64) ? ~0ull : ((1ull << avail) - 1);
            v = w << (n - avail);
        }
        b->bitpos = lo;
        return (uint32_t)(v & ((n == 32) ? 0xFFFFFFFFu : ((1u << n) - 1)));
    }
    size_t byte = (size_t)(lo >> 3); int sh = (int)(lo & 7);
    int need = (sh + n + 7) >> 3;
    for (int i = 0; i < need; i++) v |= (uint64_t)b->p[byte + (size_t)i] << (8 * i);
    b->bitpos = lo;
    return (uint32_t)((v >> sh) & ((n == 32) ? 0xFFFFFFFFull : ((1ull << n) - 1)));
}
/* peek n bits without consuming, zero-filling below the start (no overflow flag) */
static uint32_t bwd_peek(const bwd_t *b, int n) { bwd_t c = *b; return bwd_read(&c, n); }

/* ---------------------------------------------------------------- FSE */
typedef struct { uint16_t newState; uint8_t symbol; uint8_t nbBits; } fse_dentry;   /* generic symbol decode */

/* Parse a normalized-count header. Returns bytes consumed, or 0 on error. */
static size_t fse_read_ncount(int16_t *norm, uint32_t *maxSym, uint32_t *tableLog, const uint8_t *src, size_t srcSize, uint32_t maxLog) {
    fwd_t b = { src, srcSize, 0 };
    if (srcSize < 1) return 0;
    uint32_t al = fwd_peek(&b, 4) + 5; b.bitpos += 4;
    if (al > maxLog) return 0;
    int32_t remaining = 1 << al;
    uint32_t sym = 0, limit = *maxSym;
    while (remaining > 0 && sym <= limit) {
        int nb = (int)zf_highbit32((uint32_t)remaining + 1) + 1;
        uint32_t T = 1u << (nb - 1);
        uint32_t max = 2 * T - 1 - ((uint32_t)remaining + 1);
        uint32_t bits = fwd_peek(&b, nb);
        uint32_t count;
        if ((bits & (T - 1)) < max) { count = bits & (T - 1); b.bitpos += (size_t)(nb - 1); }
        else { count = bits & (2 * T - 1); if (count >= T) count -= max; b.bitpos += (size_t)nb; }
        int32_t proba = (int32_t)count - 1;
        remaining -= proba < 0 ? 1 : proba;
        norm[sym++] = (int16_t)proba;
        if (proba == 0) {
            uint32_t rep;
            do {
                rep = fwd_peek(&b, 2); b.bitpos += 2;
                for (uint32_t i = 0; i < rep; i++) { if (sym > limit) return 0; norm[sym++] = 0; }
            } while (rep == 3);
        }
        if ((b.bitpos >> 3) > srcSize + 1) return 0;
    }
    if (remaining != 0) return 0;
    if (sym == 0) return 0;
    size_t used = (b.bitpos + 7) >> 3;
    if (used > srcSize) return 0;
    *maxSym = sym - 1; *tableLog = al;
    return used;
}

static int fse_build_dtable(fse_dentry *dt, const int16_t *norm, uint32_t maxSym, uint32_t tableLog) {
    uint32_t size = 1u << tableLog, mask = size - 1, high = size - 1;
    uint16_t next[256];
    for (uint32_t s = 0; s <= maxSym; s++) {
        if (norm[s] == -1) { dt[high--].symbol = (uint8_t)s; next[s] = 1; }
        else next[s] = (uint16_t)norm[s];
    }
    uint32_t step = (size >> 1) + (size >> 3) + 3, pos = 0;
    for (uint32_t s = 0; s <= maxSym; s++)
        for (int i = 0; i < norm[s]; i++) {
            dt[pos].symbol = (uint8_t)s;
            pos = (pos + step) & mask;
            while (pos > high) pos = (pos + step) & mask;
        }
    if (pos != 0) return -1;
    for (uint32_t u = 0; u < size; u++) {
        uint32_t s = dt[u].symbol, ns = next[s]++;
        dt[u].nbBits = (uint8_t)(tableLog - zf_highbit32(ns));
        dt[u].newState = (uint16_t)((ns << dt[u].nbBits) - size);
    }
    return 0;
}

/* ---------------------------------------------------------------- Huffman */
typedef struct { uint8_t symbol, nbBits; } huf_dentry;
typedef struct { huf_dentry t[1 << ZF_HUF_MAXBITS]; uint32_t maxBits; int valid; } huf_dtable;

/* Read a Huffman tree description; returns bytes consumed or 0 on error. */
static size_t huf_read_table(huf_dtable *h, const uint8_t *src, size_t srcSize) {
    uint8_t w[256]; uint32_t nw = 0;
    if (srcSize < 1) return 0;
    uint32_t hb = src[0]; size_t used;
    if (hb >= 128) {                                      /* raw 4-bit weights */
        nw = hb - 127; used = 1 + (nw + 1) / 2;
        if (used > srcSize) return 0;
        for (uint32_t i = 0; i < nw; i++) w[i] = (i & 1) ? (src[1 + i / 2] & 15) : (src[1 + i / 2] >> 4);
    } else {                                              /* FSE-compressed weights, 2 interleaved states */
        used = 1 + hb;
        if (hb == 0 || used > srcSize) return 0;
        int16_t norm[256]; uint32_t maxSym = 255, al;
        size_t hs = fse_read_ncount(norm, &maxSym, &al, src + 1, hb, 6);
        if (!hs || hs >= hb) return 0;
        fse_dentry dt[64];
        if (fse_build_dtable(dt, norm, maxSym, al)) return 0;
        bwd_t b; if (bwd_init(&b, src + 1 + hs, hb - hs)) return 0;
        uint32_t s1 = bwd_read(&b, (int)al), s2 = bwd_read(&b, (int)al);
        if (b.overflow) return 0;
        for (;;) {
            if (nw > 253) return 0;
            w[nw++] = dt[s1].symbol; s1 = dt[s1].newState + bwd_read(&b, dt[s1].nbBits);
            if (b.overflow) { w[nw++] = dt[s2].symbol; break; }
            if (nw > 253) return 0;
            w[nw++] = dt[s2].symbol; s2 = dt[s2].newState + bwd_read(&b, dt[s2].nbBits);
            if (b.overflow) { w[nw++] = dt[s1].symbol; break; }
        }
    }
    uint32_t sum = 0, rank[ZF_HUF_MAXBITS + 2] = { 0 };
    for (uint32_t i = 0; i < nw; i++) { if (w[i] > ZF_HUF_MAXBITS) return 0; if (w[i]) sum += 1u << (w[i] - 1); }
    if (sum == 0) return 0;
    uint32_t maxBits = zf_highbit32(sum) + 1;
    if (maxBits > ZF_HUF_MAXBITS) return 0;
    uint32_t rest = (1u << maxBits) - sum;
    if (rest & (rest - 1)) return 0;                      /* must be a power of two */
    w[nw++] = (uint8_t)(zf_highbit32(rest) + 1);
    for (uint32_t i = 0; i < nw; i++) rank[w[i]]++;
    if (rank[1] < 2 || (rank[1] & 1)) return 0;
    uint32_t start[ZF_HUF_MAXBITS + 2], pos = 0;
    for (uint32_t r = 1; r <= maxBits; r++) { start[r] = pos; pos += rank[r] << (r - 1); }
    for (uint32_t s = 0; s < nw; s++) {
        uint32_t r = w[s]; if (!r) continue;
        uint32_t len = 1u << (r - 1);
        for (uint32_t i = 0; i < len; i++) { h->t[start[r] + i].symbol = (uint8_t)s; h->t[start[r] + i].nbBits = (uint8_t)(maxBits + 1 - r); }
        start[r] += len;
    }
    h->maxBits = maxBits; h->valid = 1;
    return used;
}

static int huf_decode_stream(uint8_t *dst, size_t n, const uint8_t *src, size_t srcSize, const huf_dtable *h) {
    bwd_t b; if (bwd_init(&b, src, srcSize)) return -1;
    for (size_t i = 0; i < n; i++) {
        uint32_t idx = bwd_peek(&b, (int)h->maxBits);
        dst[i] = h->t[idx].symbol;
        b.bitpos -= h->t[idx].nbBits;
    }
    return b.bitpos == 0 ? 0 : -1;
}

/* ---------------------------------------------------------------- frame state */
typedef struct { uint32_t base; uint8_t nbAdd; uint8_t nbBits; uint16_t newState; } seq_dentry;
typedef struct { seq_dentry t[512]; uint32_t log; int valid; } seq_dtable;

typedef struct {
    huf_dtable huf;
    seq_dtable ll, of, ml;
    uint32_t rep[3];
    uint8_t *lit;                                          /* ZF_BLOCK_MAX scratch */
} frame_ctx;

static int build_seq_table(seq_dtable *t, const int16_t *norm, uint32_t maxSym, uint32_t log,
                           const uint32_t *base, const uint8_t *bits) {
    fse_dentry dt[512];
    if (fse_build_dtable(dt, norm, maxSym, log)) return -1;
    for (uint32_t u = 0; u < (1u << log); u++) {
        uint32_t s = dt[u].symbol;
        t->t[u].base = base ? base[s] : (1u << s);   /* offsets: base = 1<<code, extra = code bits */
        t->t[u].nbAdd = base ? bits[s] : (uint8_t)s;
        t->t[u].nbBits = dt[u].nbBits; t->t[u].newState = dt[u].newState;
    }
    t->log = log; t->valid = 1;
    return 0;
}

/* mode: 0 predefined, 1 RLE, 2 FSE, 3 repeat. Returns bytes consumed (may be 0) or -1. */
static int64_t read_seq_table(seq_dtable *t, int mode, const uint8_t *src, size_t srcSize, uint32_t maxSymAllowed,
                              uint32_t maxLog, const int16_t *defNorm, uint32_t defMaxSym, uint32_t defLog,
                              const uint32_t *base, const uint8_t *bits) {
    if (mode == 0) return build_seq_table(t, defNorm, defMaxSym, defLog, base, bits) ? -1 : 0;
    if (mode == 1) {
        if (srcSize < 1 || src[0] > maxSymAllowed) return -1;
        uint32_t s = src[0];
        t->t[0].base = base ? base[s] : (1u << s); t->t[0].nbAdd = base ? bits[s] : (uint8_t)s;
        t->t[0].nbBits = 0; t->t[0].newState = 0; t->log = 0; t->valid = 1;
        return 1;
    }
    if (mode == 2) {
        int16_t norm[64]; uint32_t maxSym = maxSymAllowed, log;
        size_t used = fse_read_ncount(norm, &maxSym, &log, src, srcSize, maxLog);
        if (!used) return -1;
        if (build_seq_table(t, norm, maxSym, log, base, bits)) return -1;
        return (int64_t)used;
    }
    return t->valid ? 0 : -1;
}

/* Decode one compressed block. `dst` points at the block's output position, `dstStart` at the
 * start of the frame's output (history = everything before dst in this frame). */
static int64_t decode_block(frame_ctx *c, uint8_t *dst, size_t dstCap, const uint8_t *dstStart,
                            const uint8_t *src, size_t srcSize, size_t windowSize) {
    if (srcSize < 1) return -1;
    /* ---- literals section */
    uint32_t ltype = src[0] & 3, sf = (src[0] >> 2) & 3;
    size_t regen, csize = 0, hdr; int streams = 1;
    if (ltype <= 1) {
        if (sf == 0 || sf == 2) { regen = src[0] >> 3; hdr = 1; }
        else if (sf == 1) { if (srcSize < 2) return -1; regen = (src[0] >> 4) + ((size_t)src[1] << 4); hdr = 2; }
        else { if (srcSize < 3) return -1; regen = (src[0] >> 4) + ((size_t)src[1] << 4) + ((size_t)src[2] << 12); hdr = 3; }
    } else {
        if (srcSize < 5) return -1;                        /* reference requires >= MIN_CBLOCK_SIZE-ish */
        if (sf == 0 || sf == 1) { uint32_t v = src[0] | (src[1] << 8) | (src[2] << 16);
            regen = (v >> 4) & 0x3FF; csize = (v >> 14) & 0x3FF; hdr = 3; streams = sf == 0 ? 1 : 4; }
        else if (sf == 2) { uint32_t v = rd32(src); regen = (v >> 4) & 0x3FFF; csize = v >> 18; hdr = 4; streams = 4; }
        else { uint64_t v = rd32(src) | ((uint64_t)src[4] << 32); regen = (v >> 4) & 0x3FFFF; csize = (size_t)(v >> 22); hdr = 5; streams = 4; }
    }
    if (regen > ZF_BLOCK_MAX) return -1;
    const uint8_t *lit; size_t pos = hdr;
    if (ltype == 0) { if (pos + regen > srcSize) return -1; lit = src + pos; pos += regen; }
    else if (ltype == 1) { if (pos + 1 > srcSize) return -1; memset(c->lit, src[pos], regen); lit = c->lit; pos += 1; }
    else {
        if (pos + csize > srcSize) return -1;
        const uint8_t *hs = src + pos; size_t hsz = csize;
        if (ltype == 2) { size_t u = huf_read_table(&c->huf, hs, hsz); if (!u) return -1; hs += u; hsz -= u; }
        else if (!c->huf.valid) return -1;
        if (streams == 1) { if (huf_decode_stream(c->lit, regen, hs, hsz, &c->huf)) return -1; }
        else {
            if (hsz < 6) return -1;
            size_t s1 = hs[0] | (hs[1] << 8), s2 = hs[2] | (hs[3] << 8), s3 = hs[4] | (hs[5] << 8);
            if (6 + s1 + s2 + s3 > hsz) return -1;
            size_t s4 = hsz - 6 - s1 - s2 - s3, seg = (regen + 3) / 4;
            if (seg * 3 > regen) return -1;
            const uint8_t *p = hs + 6;
            if (huf_decode_stream(c->lit, seg, p, s1, &c->huf)) return -1;
            p += s1;
            if (huf_decode_stream(c->lit + seg, seg, p, s2, &c->huf)) return -1;
            p += s2;
            if (huf_decode_stream(c->lit + 2 * seg, seg, p, s3, &c->huf)) return -1;
            p += s3;
            if (huf_decode_stream(c->lit + 3 * seg, regen - 3 * seg, p, s4, &c->huf)) return -1;
        }
        lit = c->lit; pos += csize;
    }
    /* ---- sequences section */
    if (pos >= srcSize) return -1;
    uint32_t nbSeq = src[pos++];
    if (nbSeq >= 128) {
        if (nbSeq == 255) { if (pos + 2 > srcSize) return -1; nbSeq = src[pos] + (src[pos + 1] << 8) + 0x7F00; pos += 2; }
        else { if (pos + 1 > srcSize) return -1; nbSeq = ((nbSeq - 128) << 8) + src[pos++]; }
    }
    uint8_t *op = dst, *oend = dst + dstCap;
    if (nbSeq == 0) {
        if (pos != srcSize) return -1;
        if (regen > dstCap) return -2;
        memcpy(op, lit, regen);
        return (int64_t)regen;
    }
    if (pos >= srcSize) return -1;
    uint32_t modes = src[pos++];
    if (modes & 3) return -1;
    int64_t u;
    u = read_seq_table(&c->ll, modes >> 6, src + pos, srcSize - pos, ZF_MAXLL, ZF_LL_FSELOG, ZF_LL_defaultNorm, 35, ZF_LL_DEFLOG, ZF_LL_base, ZF_LL_bits);
    if (u < 0) return -1;
    pos += (size_t)u;
    u = read_seq_table(&c->of, (modes >> 4) & 3, src + pos, srcSize - pos, ZF_MAXOFF, ZF_OF_FSELOG, ZF_OF_defaultNorm, 28, ZF_OF_DEFLOG, NULL, NULL);
    if (u < 0) return -1;
    pos += (size_t)u;
    u = read_seq_table(&c->ml, (modes >> 2) & 3, src + pos, srcSize - pos, ZF_MAXML, ZF_ML_FSELOG, ZF_ML_defaultNorm, 52, ZF_ML_DEFLOG, ZF_ML_base, ZF_ML_bits);
    if (u < 0) return -1;
    pos += (size_t)u;
    bwd_t b; if (bwd_init(&b, src + pos, srcSize - pos)) return -1;
    uint32_t sLL = bwd_read(&b, (int)c->ll.log), sOF = bwd_read(&b, (int)c->of.log), sML = bwd_read(&b, (int)c->ml.log);
    if (b.overflow) return -1;
    const uint8_t *lp = lit, *lend = lit + regen;
    for (uint32_t i = 0; i < nbSeq; i++) {
        const seq_dentry *eL = &c->ll.t[sLL], *eO = &c->of.t[sOF], *eM = &c->ml.t[sML];
        uint32_t offBase = eO->base + bwd_read(&b, eO->nbAdd);
        uint32_t ml = eM->base + bwd_read(&b, eM->nbAdd);
        uint32_t ll = eL->base + bwd_read(&b, eL->nbAdd);
        uint32_t offset;
        if (eO->nbAdd > 1 || offBase > 3) {               /* codes >= 2 (offBase >= 4) are real offsets */
            offset = offBase - 3; c->rep[2] = c->rep[1]; c->rep[1] = c->rep[0]; c->rep[0] = offset;
        } else {
            uint32_t idx = offBase - 1 + (ll == 0);        /* offBase in 1..3 */
            if (idx == 0) offset = c->rep[0];
            else {
                offset = idx == 3 ? c->rep[0] - 1 : c->rep[idx];
                if (offset == 0) return -1;                /* reference maps 0 -> corruption */
                if (idx != 1) c->rep[2] = c->rep[1];
                c->rep[1] = c->rep[0]; c->rep[0] = offset;
            }
        }
        if (i + 1 < nbSeq) {
            sLL = eL->newState + bwd_read(&b, eL->nbBits);
            sML = eM->newState + bwd_read(&b, eM->nbBits);
            sOF = eO->newState + bwd_read(&b, eO->nbBits);
        }
        if (b.overflow) return -1;
        if ((size_t)(lend - lp) < ll) return -1;
        if ((size_t)(oend - op) < (size_t)ll + ml) return -2;
        memcpy(op, lp, ll); op += ll; lp += ll;
        if (offset > (size_t)(op - dstStart) || offset > windowSize) return -1;
        const uint8_t *m = op - offset;
        for (uint32_t k = 0; k < ml; k++) op[k] = m[k];   /* byte-wise: overlap-safe */
        op += ml;
    }
    if (b.bitpos != 0) return -1;
    size_t tail = (size_t)(lend - lp);
    if ((size_t)(oend - op) < tail) return -2;
    memcpy(op, lp, tail); op += tail;
    return (int64_t)(op - dst);
}

/* Decode all frames in [src, src+srcSize). Returns decompressed size, or a negative error:
 * -1 corrupt, -2 dst too small, -3 checksum mismatch, -4 unsupported (dictionary). */
int64_t b2zo_zstd_decompress(void *dstv, size_t dstCap, const void *srcv, size_t srcSize) {
    const uint8_t *src = (const uint8_t *)srcv, *ip = src, *iend = src + srcSize;
    uint8_t *dst = (uint8_t *)dstv, *op = dst, *oend = dst + dstCap;
    frame_ctx *c = (frame_ctx *)malloc(sizeof(frame_ctx));
    uint8_t *litbuf = (uint8_t *)malloc(ZF_BLOCK_MAX + 32);
    int64_t rc = 0;
    while (ip < iend) {
        if (iend - ip < 4) { rc = -1; break; }
        uint32_t magic = rd32(ip);
        if ((magic & ZF_MAGIC_SKIP_MASK) == ZF_MAGIC_SKIP) {
            if (iend - ip < 8) { rc = -1; break; }
            uint32_t sz = rd32(ip + 4);
            if ((size_t)(iend - ip) < 8 + (size_t)sz) { rc = -1; break; }
            ip += 8 + sz; continue;
        }
        if (magic != ZF_MAGIC) { rc = -1; break; }
        if (iend - ip < 6) { rc = -1; break; }
        uint32_t fhd = ip[4]; ip += 5;
        uint32_t fcsFlag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, didFlag = fhd & 3;
        if (fhd & 8) { rc = -1; break; }
        uint64_t windowSize = 0, fcs = ~0ull;
        if (!single) { uint32_t wd = *ip++; uint32_t wl = 10 + (wd >> 3); if (wl > 31) { rc = -1; break; }
            windowSize = (1ull << wl) + ((1ull << wl) >> 3) * (wd & 7); }
        static const int didBytes[4] = { 0, 1, 2, 4 };
        if (iend - ip < didBytes[didFlag]) { rc = -1; break; }
        uint32_t did = 0; for (int i = 0; i < didBytes[didFlag]; i++) did |= (uint32_t)ip[i] << (8 * i);
        ip += didBytes[didFlag];
        if (did) { rc = -4; break; }
        int fcsBytes = fcsFlag == 0 ? (int)single : (fcsFlag == 1 ? 2 : (fcsFlag == 2 ? 4 : 8));
        if (iend - ip < fcsBytes) { rc = -1; break; }
        if (fcsBytes) { fcs = 0; for (int i = 0; i < fcsBytes; i++) fcs |= (uint64_t)ip[i] << (8 * i); if (fcsBytes == 2) fcs += 256; }
        ip += fcsBytes;
        if (single) windowSize = fcs;
        memset(c, 0, sizeof(*c)); c->lit = litbuf;
        c->rep[0] = 1; c->rep[1] = 4; c->rep[2] = 8;
        uint8_t *frameStart = op;
        size_t blockMax = windowSize < ZF_BLOCK_MAX ? (size_t)windowSize : ZF_BLOCK_MAX;
        for (;;) {
            if (iend - ip < 3) { rc = -1; goto done; }
            uint32_t bh = ip[0] | (ip[1] << 8) | (ip[2] << 16); ip += 3;
            uint32_t last = bh & 1, type = (bh >> 1) & 3, bsize = bh >> 3;
            if (bsize > blockMax) { rc = -1; goto done; }      /* RFC 8878 3.1.1.2.4: Block_Maximum_Size = min(Window_Size, 128 KiB) */
            if (type == 0) {
                if ((size_t)(iend - ip) < bsize) { rc = -1; goto done; }
                if ((size_t)(oend - op) < bsize) { rc = -2; goto done; }
                if (bsize > ZF_BLOCK_MAX) { rc = -1; goto done; }
                memcpy(op, ip, bsize); op += bsize; ip += bsize;
            } else if (type == 1) {
                if (iend - ip < 1) { rc = -1; goto done; }
                if ((size_t)(oend - op) < bsize) { rc = -2; goto done; }
                if (bsize > ZF_BLOCK_MAX) { rc = -1; goto done; }
                memset(op, *ip, bsize); op += bsize; ip += 1;
            } else if (type == 2) {
                if ((size_t)(iend - ip) < bsize || bsize > ZF_BLOCK_MAX) { rc = -1; goto done; }
                size_t cap = (size_t)(oend - op) < ZF_BLOCK_MAX ? (size_t)(oend - op) : ZF_BLOCK_MAX;
                int64_t r = decode_block(c, op, cap, frameStart, ip, bsize, (size_t)windowSize);
                if (r < 0) { rc = ((size_t)(oend - op) < ZF_BLOCK_MAX && r == -2) ? -2 : (r == -2 ? -1 : r); goto done; }
                if ((size_t)r > blockMax) { rc = -1; goto done; }  /* nor may a compressed block decode to more */
                op += r; ip += bsize;
            } else { rc = -1; goto done; }
            if (last) break;
        }
        if (fcs != ~0ull && (uint64_t)(op - frameStart) != fcs) { rc = -1; break; }
        if (checksum) {
            if (iend - ip < 4) { rc = -1; break; }
            uint32_t want = rd32(ip); ip += 4;
            if ((uint32_t)b2zo_xxh64(frameStart, (size_t)(op - frameStart), 0) != want) { rc = -3; break; }
        }
    }
done:
    free(litbuf); free(c);
    return rc < 0 ? rc : (int64_t)(op - dst);
}
