/* lzma2_enc_oracle.c -- sequential statement of the GPU LZMA2 encoder (7-Zip method 21).
 *
 * TEST INFRASTRUCTURE ONLY (see oracle.h).  The encoder's byte stream is ours (the reference pins no encoder bytes,
 * SURVEY.md 8c); what is pinned: the reference decoder (C/Lzma2Dec.c via oracle/_ref), liblzma and the oracle decoder all
 * restore the input from it, and the GPU must produce exactly these bytes.
 *
 * Shape: the input is cut into frames of 2^frameLog bytes; each frame becomes one dictionary-reset LZMA2 block (the unit
 * the reference's own MT coders use, Lzma2Enc.c:241-330 block split, Lzma2DecMt.c:237).  Inside a frame:
 *   stage M  the match finder / greedy-lazy parser shared with the zstd path (find_sequences of zstd_enc_oracle.c)
 *            -- or, with flag B2Z_FLAG_LZ2_OPT, stage C + stage P: candidates and the price-based parse (lzma2_opt_oracle.c)
 *   stage R  this file: the sequences are coded as LZMA packets (literal / match / rep0-3) with the adaptive binary range
 *            coder, cut into LZMA2 chunks, with the raw-chunk fallback for chunks that do not shrink.
 *
 * Reference functions whose format rules are followed (under /root/reference/C/):
 *   range coder: RangeEnc_ShiftLow / RC_BIT ......... LzmaEnc.c:691-760 ; fast-lzma2/range_enc.c:123-197
 *   literal / matched literal ........................ LzmaEnc.c:795-860 (LitEnc_Encode, LitEnc_EncodeMatched)
 *   length coder ..................................... LzmaEnc.c:934-1010 (LenEnc_Encode)
 *   match / rep packets, distance slots, align bits .. LzmaEnc.c:2388-2600 (LzmaEnc_CodeOneBlock)
 *   chunk headers, props byte, copy-chunk fallback ... Lzma2Enc.c:129-238 (Lzma2EncInt_EncodeSubblock); fast-lzma2/lzma2_enc.c:1937-2099
 */
#include <stdlib.h>
#include <string.h>
#include "oracle.h"
#include "b2z_params.h"

#define kNumStates 12
#define PROB_INIT 1024
#define kTop (1u << 24)

enum { P_ISMATCH = 0, P_ISREP = 192, P_ISREPG0 = 204, P_ISREPG1 = 216, P_ISREPG2 = 228, P_ISREP0LONG = 240, P_POSSLOT = 432,
       P_SPECPOS = 688, P_ALIGN = 804, P_LEN = 820, P_REPLEN = 1334, P_LIT = 1848,
       L_CHOICE = 0, L_CHOICE2 = 1, L_LOW = 2, L_MID = 130, L_HIGH = 258 };

typedef struct {
    uint16_t probs[P_LIT + (0x300 << (B2Z_LZ2_LC + B2Z_LZ2_LP))];
    uint32_t state, rep[4];
    uint64_t low; uint32_t range, cacheSize; uint8_t cache;
    uint8_t *out; size_t op;
    uint32_t modelResets;                /* chunk_open calls that initialised the model (test tap) */
} enc_t;

static void rc_shift_low(enc_t *e) {
    if ((uint32_t)e->low < 0xFF000000u || (uint32_t)(e->low >> 32) != 0) {
        const uint8_t carry = (uint8_t)(e->low >> 32);
        uint8_t c = e->cache;
        do { e->out[e->op++] = (uint8_t)(c + carry); c = 0xFF; } while (--e->cacheSize != 0);
        e->cache = (uint8_t)((uint32_t)e->low >> 24);
    }
    e->cacheSize++;
    e->low = (e->low & 0x00FFFFFFu) << 8;
}
static void rc_bit(enc_t *e, uint16_t *p, uint32_t bit) {
    const uint32_t v = *p, bound = (e->range >> 11) * v;
    if (!bit) { e->range = bound; *p = (uint16_t)(v + ((2048 - v) >> 5)); }
    else { e->low += bound; e->range -= bound; *p = (uint16_t)(v - (v >> 5)); }
    while (e->range < kTop) { e->range <<= 8; rc_shift_low(e); }
}
static void rc_direct(enc_t *e, uint32_t v, uint32_t n) {
    while (n--) { e->range >>= 1; if ((v >> n) & 1) e->low += e->range; while (e->range < kTop) { e->range <<= 8; rc_shift_low(e); } }
}
static void rc_tree(enc_t *e, uint16_t *p, uint32_t bits, uint32_t v) { uint32_t m = 1; for (uint32_t i = bits; i--;) { uint32_t b = (v >> i) & 1; rc_bit(e, p + m, b); m = (m << 1) | b; } }
static void rc_tree_rev(enc_t *e, uint16_t *p, uint32_t bits, uint32_t v) { uint32_t m = 1; for (uint32_t i = 0; i < bits; i++) { uint32_t b = (v >> i) & 1; rc_bit(e, p + m, b); m = (m << 1) | b; } }
static void rc_len(enc_t *e, uint16_t *l, uint32_t len, uint32_t ps) {
    len -= 2;
    if (len < 8) { rc_bit(e, l + L_CHOICE, 0); rc_tree(e, l + L_LOW + ps * 8, 3, len); }
    else if (len < 16) { rc_bit(e, l + L_CHOICE, 1); rc_bit(e, l + L_CHOICE2, 0); rc_tree(e, l + L_MID + ps * 8, 3, len - 8); }
    else { rc_bit(e, l + L_CHOICE, 1); rc_bit(e, l + L_CHOICE2, 1); rc_tree(e, l + L_HIGH, 8, len - 16); }
}

static void enc_literal(enc_t *e, const uint8_t *base, uint32_t pos) {
    const uint32_t ps = pos & ((1u << B2Z_LZ2_PB) - 1), prev = pos ? base[pos - 1] : 0, sym = base[pos];
    rc_bit(e, e->probs + P_ISMATCH + e->state * 16 + ps, 0);
    uint16_t *p = e->probs + P_LIT + 0x300 * (((pos & ((1u << B2Z_LZ2_LP) - 1)) << B2Z_LZ2_LC) + (prev >> (8 - B2Z_LZ2_LC)));
    uint32_t m = 1; int matched = e->state >= 7;
    const uint32_t mb = matched ? base[pos - e->rep[0] - 1] : 0;
    for (uint32_t i = 8; i--;) {
        const uint32_t b = (sym >> i) & 1;
        if (matched) { const uint32_t mbit = (mb >> i) & 1; rc_bit(e, p + ((1 + mbit) << 8) + m, b); if (mbit != b) matched = 0; }
        else rc_bit(e, p + m, b);
        m = (m << 1) | b;
    }
    e->state = e->state < 4 ? 0 : (e->state < 10 ? e->state - 3 : e->state - 6);
}

/* one match packet of len (2..273) at distance dist1 (= distance - 1) */
static void enc_match(enc_t *e, uint32_t pos, uint32_t len, uint32_t dist) {
    const uint32_t ps = pos & ((1u << B2Z_LZ2_PB) - 1);
    rc_bit(e, e->probs + P_ISMATCH + e->state * 16 + ps, 1);
    int r = -1;
    for (int i = 0; i < 4; i++) if (e->rep[i] == dist) { r = i; break; }
    if (r >= 0 && pos == 0) r = -1;
    if (r < 0) {
        rc_bit(e, e->probs + P_ISREP + e->state, 0);
        rc_len(e, e->probs + P_LEN, len, ps);
        e->state = e->state < 7 ? 7 : 10;
        uint32_t slot;
        if (dist < 4) slot = dist; else { uint32_t nb = 31 - (uint32_t)__builtin_clz(dist); slot = (nb << 1) | ((dist >> (nb - 1)) & 1); }
        rc_tree(e, e->probs + P_POSSLOT + (len - 2 < 4 ? len - 2 : 3) * 64, 6, slot);
        if (slot >= 4) {
            const uint32_t fb = (slot >> 1) - 1, b = (2 | (slot & 1)) << fb, red = dist - b;
            if (slot < 14) rc_tree_rev(e, e->probs + P_SPECPOS + b - slot - 1, fb, red);
            else { rc_direct(e, red >> 4, fb - 4); rc_tree_rev(e, e->probs + P_ALIGN, 4, red & 15); }
        }
        e->rep[3] = e->rep[2]; e->rep[2] = e->rep[1]; e->rep[1] = e->rep[0]; e->rep[0] = dist;
    } else {
        rc_bit(e, e->probs + P_ISREP + e->state, 1);
        if (r == 0) { rc_bit(e, e->probs + P_ISREPG0 + e->state, 0); rc_bit(e, e->probs + P_ISREP0LONG + e->state * 16 + ps, 1); }
        else {
            rc_bit(e, e->probs + P_ISREPG0 + e->state, 1);
            if (r == 1) rc_bit(e, e->probs + P_ISREPG1 + e->state, 0);
            else { rc_bit(e, e->probs + P_ISREPG1 + e->state, 1); rc_bit(e, e->probs + P_ISREPG2 + e->state, (uint32_t)(r - 2)); }
            for (int i = r; i > 0; i--) e->rep[i] = e->rep[i - 1];
            e->rep[0] = dist;
        }
        rc_len(e, e->probs + P_REPLEN, len, ps);
        e->state = e->state < 7 ? 8 : 11;
    }
}

/* chunk bookkeeping of one frame */
typedef struct { enc_t *e; const uint8_t *base; uint32_t chunkPos, chunkOut, hdr; int open, needDict, needProps, needState; } chunker;

static void chunk_open(chunker *c, uint32_t pos) {
    enc_t *e = c->e;
    c->chunkPos = pos; c->chunkOut = (uint32_t)e->op;
    c->hdr = (c->needDict || c->needProps) ? 6 : 5;
    if (c->needDict || c->needProps || c->needState) {
        for (size_t i = 0; i < sizeof(e->probs) / 2; i++) e->probs[i] = PROB_INIT;
        e->modelResets++;
        e->state = 0; e->rep[0] = e->rep[1] = e->rep[2] = e->rep[3] = 0;
    }
    e->op += c->hdr;
    e->low = 0; e->range = 0xFFFFFFFFu; e->cache = 0; e->cacheSize = 1;
    c->open = 1;
}
static void chunk_close(chunker *c, uint32_t pos) {
    enc_t *e = c->e;
    if (!c->open) return;
    for (int i = 0; i < 5; i++) rc_shift_low(e);
    const uint32_t unpack = pos - c->chunkPos, pack = (uint32_t)e->op - c->chunkOut - c->hdr;
    uint8_t *h = e->out + c->chunkOut;
    if (pack + 2 >= unpack) {                                   /* Lzma2Enc.c:183-185: store the chunk uncompressed */
        h[0] = c->needDict ? 1 : 2; h[1] = (uint8_t)((unpack - 1) >> 8); h[2] = (uint8_t)(unpack - 1);
        memcpy(h + 3, c->base + c->chunkPos, unpack);
        e->op = c->chunkOut + 3 + unpack;
        c->needDict = 0; c->needState = 1;
    } else {
        const uint32_t mode = c->needDict ? 3 : (c->needProps ? 2 : (c->needState ? 1 : 0));
        h[0] = (uint8_t)(0x80 | (mode << 5) | ((unpack - 1) >> 16)); h[1] = (uint8_t)((unpack - 1) >> 8); h[2] = (uint8_t)(unpack - 1);
        h[3] = (uint8_t)((pack - 1) >> 8); h[4] = (uint8_t)(pack - 1);
        if (mode >= 2) h[5] = (uint8_t)B2Z_LZ2_PROPS;
        c->needDict = c->needProps = c->needState = 0;
    }
    c->open = 0;
}
/* before every packet: open a chunk if none, or roll over to a new one when a limit is reached */
static void chunk_step(chunker *c, uint32_t pos) {
    enc_t *e = c->e;
    if (c->open && ((uint32_t)e->op - c->chunkOut - c->hdr + e->cacheSize >= B2Z_LZ2_PACK_LIMIT || pos - c->chunkPos >= B2Z_LZ2_UNPACK_LIMIT)) chunk_close(c, pos);
    if (!c->open) chunk_open(c, pos);
}

/* sliceBlocks: a frame is coded as slices of this many 128 KiB blocks; every slice after the first starts a new chunk with a
 * state reset (control 0xA0: fresh model, same dictionary), which makes the slices' range coders independent of each other --
 * the scheme of fast-lzma2's encoder threads (lzma2_enc.c:1937-2099 "props/state reset at slice start") */
static size_t encode_frame(enc_t *e, const uint8_t *base, uint32_t n, const uint64_t *seqs, const uint32_t *nseq, uint8_t *out, uint32_t sliceBlocks) {
    chunker c; memset(&c, 0, sizeof(c));
    c.e = e; c.base = base; c.needDict = c.needProps = c.needState = 1;
    e->out = out; e->op = 0;
    const uint32_t nblk = (n + B2Z_BLOCK - 1) / B2Z_BLOCK;
    uint32_t pos = 0;
    for (uint32_t b = 0; b < nblk; b++) {
        const uint32_t bend = (b + 1) * B2Z_BLOCK < n ? (b + 1) * B2Z_BLOCK : n;
        if (b && b % sliceBlocks == 0) { chunk_close(&c, pos); c.needState = c.needProps = 1; }   /* a slice never depends on what the previous one emitted */
        uint32_t zr[3] = {0, 0, 0};                             /* zstd repcode history of the block (0 = unknown), to undo offBase */
        for (uint32_t i = 0; i < nseq[b]; i++) {
            const uint64_t s = seqs[(size_t)b * B2Z_MAXSEQ + i];
            const uint32_t ll = B2Z_SEQ_LL(s), ob = B2Z_SEQ_OFFBASE(s); uint32_t ml = B2Z_SEQ_ML(s), off;
            if (ob > 3) { off = ob - 3; zr[2] = zr[1]; zr[1] = zr[0]; zr[0] = off; }
            else {
                const uint32_t idx = ob - 1 + (ll == 0);
                off = idx == 3 ? zr[0] - 1 : zr[idx];
                if (idx != 0) { if (idx != 1) zr[2] = zr[1]; zr[1] = zr[0]; zr[0] = off; }
            }
            for (uint32_t j = 0; j < ll; j++) { chunk_step(&c, pos); enc_literal(e, base, pos); pos++; }
            while (ml) {
                uint32_t len = ml > B2Z_LZ2_MAXLEN ? B2Z_LZ2_MAXLEN : ml;
                if (ml - len == 1) len--;                       /* never leave a 1-byte tail */
                chunk_step(&c, pos); enc_match(e, pos, len, off - 1); pos += len; ml -= len;
            }
        }
        while (pos < bend) { chunk_step(&c, pos); enc_literal(e, base, pos); pos++; }
    }
    chunk_close(&c, pos);
    return e->op;
}

/* Test tap: the model stage R ends a frame with (probabilities, state, rep0-3) after coding the given sequences, and how often it
 * initialised the model on the way (slices + raw-chunk fallbacks).  Lets tests pin stage P's simulated model (b2z_lzma_model.h:
 * lzm_commit_*) to this independent statement of the coder. */
int64_t b2zo_lzma2_final_model(const void *basev, uint32_t n, const b2zo_enc_params *P, const uint64_t *seqs, const uint32_t *nseq,
                               uint16_t *probsOut, uint32_t *ctxOut /* state, rep0..3 */) {
    enc_t *e = (enc_t *)calloc(1, sizeof(enc_t));
    uint8_t *tmp = (uint8_t *)malloc(B2Z_LZ2_FRAME_BOUND(n));
    encode_frame(e, (const uint8_t *)basev, n, seqs, nseq, tmp, B2Z_LZ2_SLICE_BLOCKS(P->frameLog, P->flags));
    memcpy(probsOut, e->probs, sizeof(e->probs));
    ctxOut[0] = e->state; for (int i = 0; i < 4; i++) ctxOut[1 + i] = e->rep[i];
    const int64_t resets = e->modelResets;
    free(tmp); free(e);
    return resets;
}

size_t b2zo_lzma2_compress_bound(size_t n, const b2zo_enc_params *p) {
    const size_t F = (size_t)1 << p->frameLog, frames = (n + F - 1) / F;
    return frames * (size_t)B2Z_LZ2_FRAME_BOUND((uint32_t)F) + 1;
}

/* -> raw LZMA2 stream (chunks + 0x00); *dictProp = the coder property a 7z folder would carry (Lzma2Enc_WriteProperties) */
int64_t b2zo_lzma2_compress(void *dstv, size_t dstCap, const void *srcv, size_t srcSize, const b2zo_enc_params *p, uint32_t *dictProp) {
    const uint8_t *src = (const uint8_t *)srcv; uint8_t *dst = (uint8_t *)dstv;
    const size_t F = (size_t)1 << p->frameLog;
    if (dictProp) *dictProp = p->frameLog >= 12 ? (p->frameLog - 12) * 2 : 0;          /* dictionary = frame size */
    size_t op = 0;
    if (srcSize) {
        const size_t nblkAll = (srcSize + B2Z_BLOCK - 1) / B2Z_BLOCK;
        uint64_t *seqs = (uint64_t *)malloc(nblkAll * B2Z_MAXSEQ * sizeof(uint64_t));
        uint32_t *nseq = (uint32_t *)calloc(nblkAll, 4), *nlit = (uint32_t *)calloc(nblkAll, 4);
        uint8_t *lits = (uint8_t *)malloc(srcSize);
        uint8_t *tmp = (uint8_t *)malloc(B2Z_LZ2_FRAME_BOUND(F));
        enc_t *e = (enc_t *)malloc(sizeof(enc_t));
        const size_t bpf = F / B2Z_BLOCK;
        if (p->flags & B2Z_FLAG_LZ2_OPT) {
            for (size_t f = 0, f0 = 0; f0 < srcSize; f++, f0 += F)
                b2zo_lzma2_parse_frame(src + f0, (uint32_t)(srcSize - f0 < F ? srcSize - f0 : F), p, NULL, seqs + f * bpf * B2Z_MAXSEQ, nseq + f * bpf);
        } else { b2zo_enc_params q = *p; q.regionLog = 0; q.ldmLog = 0;              /* method 21 has no regions: a block is stage F's unit */
                 b2zo_zstd_find_sequences(src, srcSize, &q, seqs, nseq, lits, nlit); }
        int fail = 0;
        for (size_t f = 0, f0 = 0; f0 < srcSize; f++, f0 += F) {
            const uint32_t n = (uint32_t)(srcSize - f0 < F ? srcSize - f0 : F);
            const size_t sz = encode_frame(e, src + f0, n, seqs + f * bpf * B2Z_MAXSEQ, nseq + f * bpf, tmp, B2Z_LZ2_SLICE_BLOCKS(p->frameLog, p->flags));
            if (op + sz + 1 > dstCap) { fail = 1; break; }
            memcpy(dst + op, tmp, sz); op += sz;
        }
        free(seqs); free(nseq); free(nlit); free(lits); free(tmp); free(e);
        if (fail) return -2;
    }
    if (op + 1 > dstCap) return -2;
    dst[op++] = 0;
    return (int64_t)op;
}
