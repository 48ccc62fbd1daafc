/* zstd_enc_oracle.c -- plain-C restatement of the GPU block-parallel Zstandard encoder.
 *
 * TEST INFRASTRUCTURE ONLY (see oracle.h).  This is the single-threaded statement of the
 * algorithm that 7-zip-zstd_b200/csrc/zstd_enc_*.cu implements with one CTA per frame
 * (stage F), one warp per 128 KiB block (stage G, stage E).  Every decision below is integer and
 * order-independent by construction, so the CUDA path must reproduce these bytes exactly;
 * tests compare stage taps (raw sequences, literals) and final frames byte-for-byte.
 *
 * What it replaces in the reference (level 3 = dfast; /root/reference/C/zstd/):
 *   ZSTDMT job slicing ............... zstdmt_compress.c:1184-1246  -> independent frames of 2^frameLog
 *   ZSTD_compress_frameChunk ......... zstd_compress.c:4591          -> 128 KiB blocks, 3-byte headers
 *   ZSTD_compressBlock_doubleFast .... zstd_double_fast.c:103-330    -> stage F (dual hash, all positions) + stage G (parse)
 *   ZSTD_hash5Ptr / ZSTD_hash8Ptr .... zstd_compress_internal.h:903-924 (same multiplicative hashes)
 *   ZSTD_storeSeq / ZSTD_updateRep ... zstd_compress_internal.h:775,817 -> merge + repcode pass
 *   ZSTD_compressLiterals ............ zstd_compress_literals.c:129-235
 *   HUF_buildCTable / writeCTable .... huf_compress.c:755,248        -> own length-limited builder
 *   HUF_compress4X_usingCTable ....... huf_compress.c:1167
 *   ZSTD_seqToCodes .................. zstd_compress.c:2693
 *   ZSTD_buildSequencesStatistics .... zstd_compress.c:2763; zstd_compress_sequences.c:156,242
 *   FSE_normalizeCount/writeNCount/buildCTable  fse_compress.c:465,330,68 -> own normaliser
 *   ZSTD_encodeSequences ............. zstd_compress_sequences.c:291-382
 *   ZSTD_writeFrameHeader/Epilogue ... zstd_compress.c:4695,5344
 * The encoder's OUTPUT BYTES are not pinned by the reference (SURVEY.md 4: no known-answer
 * test exists); parity = the reference decoder round-trips every frame + ratio delta.
 *
 * Parallel semantics restated sequentially:
 *   - stage F: a CTA owns a frame and walks it in chunks of 2^chunkLog positions; a position sees the tables as they
 *     stood before its chunk (b2zo_zstd_candidates);
 *   - stage G: a warp owns a 128 KiB block, a lane a 4 KiB segment of it: minimum-price path per segment, repcode
 *     history unknown at every segment start (parse_frame).
 */
#include <string.h>
#include <stdlib.h>
#include "zstd_format.h"
#include "oracle.h"
#include "b2z_params.h"
#include "b2z_zstd_cost.h"

static inline uint64_t rd64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline void wr16(uint8_t *p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
static inline void wr24(uint8_t *p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); }
static inline void wr32(uint8_t *p, uint32_t v) { memcpy(p, &v, 4); }

void b2zo_enc_default_params(b2zo_enc_params *p, int level) {
    p->frameLog = B2Z_DEF_FRAMELOG; p->hashLogL = B2Z_DEF_HASHLOG_L; p->hashLogS = B2Z_DEF_HASHLOG_S;
    p->windowLog = B2Z_DEF_FRAMELOG; p->chunkLog = B2Z_DEF_CHUNKLOG; p->flags = 1u | (B2Z_DEF_LZ2_SLICELOG << 8);
    p->regionLog = B2Z_DEF_PLAIN_REGIONLOG; p->ldmLog = 0;
    p->flags |= b2z_level_find_flags(level) | (level >= B2Z_ZSTD_OPT_LEVEL ? B2Z_FLAG_ZSTD_OPT : 0u);      /* what B200Z_P_LEVEL sets */
    if (p->flags & B2Z_FLAG_FIND_FAST) p->hashLogS = B2Z_DEF_HASHLOG_L;                                     /* the single table takes the long table's room */
}

size_t b2zo_zstd_compress_bound(size_t n, const b2zo_enc_params *p) {
    size_t frames = (n >> p->frameLog) + 1, blocks = (n >> 17) + frames;
    return n + blocks * 3 + frames * (B2Z_FRAME_HDR_MAX + 12 + 4) + 64;
}

/* ======================================================================= stage F + stage G */
static size_t count_match(const uint8_t *a, const uint8_t *b, size_t maxLen) {
    size_t n = 0;
    while (n + 8 <= maxLen) {
        uint64_t x = rd64(a + n) ^ rd64(b + n);
        if (x) return n + ((size_t)__builtin_ctzll(x) >> 3);
        n += 8;
    }
    while (n < maxLen && a[n] == b[n]) n++;
    return n;
}

/* Stage F, one frame: src[0..n) -> one candidate word per position (b2z_params.h: B2Z_CAND).
 *
 * Two direct-mapped tables of position+tag entries, the long one indexed by the 8-byte hash and the short one by the
 * 5-byte hash of the reference's double-fast finder (zstd_double_fast.c:103-330, constants zstd_compress_internal.h:903-924)
 * -- sized for the shared memory of one SM (2^15 + 2^14 entries), not for the 2^17 + 2^16 of level 3.  The frame is
 * walked in CHUNKS of 2^chunkLog positions: a position sees the tables as they stood BEFORE its chunk; after a chunk every
 * table entry holds the highest position of the chunk that indexes it.  That is a pure function of the frame's bytes: the
 * kernel evaluates a chunk with 2^chunkLog threads (reads, barrier, atomicMax writes).  (Letting a position also see the
 * lower positions of its own 32-position step costs two __match_any_sync per step -- the SM's ADU pipe became the bound --
 * and buys nothing on text: 2.3823 vs 2.3830 on G2; structured data with repeats at distances under 128 loses about 1 %.)
 * Every position is searched and inserted.  Candidates are compared over at most B2Z_CAP bytes and never beyond the end
 * of their 4 KiB parse segment; the longer of (long, short) wins, the nearer on a tie. */
static void candidates_region(const uint8_t *src, uint32_t n, const b2zo_enc_params *P, uint32_t unitLog, uint32_t *cand) {
    const uint32_t HL = P->hashLogL, HS = P->hashLogS, CH = 1u << P->chunkLog;
    const uint32_t tagBits = 32 - (unitLog + 1), tagMask = (1u << tagBits) - 1;
    const uint64_t W = P->windowLog >= 32 ? 0xFFFFFFFFull : (1ull << P->windowLog);
    const int FAST = (P->flags & B2Z_FLAG_FIND_FAST) != 0, STEP = (P->flags & B2Z_FLAG_FIND_STEP) != 0;
    uint32_t *TL = (uint32_t *)calloc((size_t)1 << HL, 4), *TS = (uint32_t *)calloc((size_t)1 << HS, 4);
    uint32_t *iL = (uint32_t *)malloc(CH * 4), *iS = (uint32_t *)malloc(CH * 4), *eLn = (uint32_t *)malloc(CH * 4), *eSn = (uint32_t *)malloc(CH * 4);
    for (uint32_t c0 = 0; c0 < n; c0 += CH) {
        const uint32_t c1 = n - c0 < CH ? n : c0 + CH;
        for (uint32_t p = c0; p < c1; p++) {
            const uint32_t k = p - c0;
            iL[k] = iS[k] = 0xFFFFFFFFu; cand[p] = 0;
            if (p + 8 > n) continue;                                            /* the last 7 positions are neither searched nor inserted */
            const uint64_t v = rd64(src + p), hl = v * B2Z_PRIME8, hs = (v << 24) * B2Z_PRIME5;
            iL[k] = (uint32_t)(hl >> (64 - HL)); iS[k] = (uint32_t)(hs >> (64 - HS));
            const uint32_t tL = (uint32_t)(hl >> (64 - HL - tagBits)) & tagMask, tS = (uint32_t)(hs >> (64 - HS - tagBits)) & tagMask;
            eLn[k] = ((p + 1) << tagBits) | tL; eSn[k] = ((p + 1) << tagBits) | tS;
            uint32_t eL = FAST ? 0u : TL[iL[k]], eS = TS[iS[k]];             /* the tables as they stood before this chunk */
            if (STEP) for (uint32_t q = p & ~31u; q < p; q++) {                /* levels 5-7: nearer, the lower positions of the same 32-position step */
                if (!FAST && iL[q - c0] == iL[k]) eL = eLn[q - c0];
                if (iS[q - c0] == iS[k]) eS = eSn[q - c0];
            }
            const uint32_t segEnd = ((p | (B2Z_SEG - 1)) + 1) < n ? ((p | (B2Z_SEG - 1)) + 1) : n;
            uint32_t maxLen = segEnd - p; if (maxLen > B2Z_CAP) maxLen = B2Z_CAP;
            uint32_t lenL = 0, offL = 0, lenS = 0, offS = 0;
            if (eL && (eL & tagMask) == tL) { const uint32_t q = (eL >> tagBits) - 1; if (p - q <= W) { offL = p - q; lenL = (uint32_t)count_match(src + q, src + p, maxLen); } }
            if (eS && (eS & tagMask) == tS) { const uint32_t q = (eS >> tagBits) - 1; if (p - q <= W && p - q != offL) { offS = p - q; lenS = (uint32_t)count_match(src + q, src + p, maxLen); } }
            uint32_t len = lenL, off = offL;
            if (lenS > lenL || (lenS == lenL && lenS && offS < offL)) { len = lenS; off = offS; }
            if (len >= B2Z_DP_MINLEN) cand[p] = B2Z_CAND(len, off);
        }
        for (uint32_t k = 0; k < c1 - c0; k++) if (iL[k] != 0xFFFFFFFFu) { TL[iL[k]] = eLn[k]; TS[iS[k]] = eSn[k]; }   /* ascending: the highest position stays */
    }
    free(TL); free(TS); free(iL); free(iS); free(eLn); free(eSn);
}

/* Stage L, one frame of the long mode (the role of zstd_ldm.c:333-470, ZSTD_ldm_generateSequences: rolling-hash split points, a
 * bucketed table of checksums, matches of >= minMatchLength 64 bytes found far behind the reach of the block finder).  Restated
 * for the device as a pure function of the frame's bytes, in two passes that are each parallel over every position:
 *   - position p is a SAMPLE when a hash of its 8 bytes has its top B2Z_LDM_RATELOG bits set (content-defined, so both ends of a
 *     far copy sample the same places); its key hashes the 32 bytes at p;
 *   - the frame is cut into EPOCHS of half a window; pass 1: one direct-mapped table per epoch, entry = position in the epoch
 *     << 4 | tag, keeps the LOWEST sample of every index (atomicMin on the device): the first occurrence in the epoch;
 *   - pass 2: a sample looks its index up in its own epoch's table and the two before it (together they cover the window), nearest
 *     first; the first entry that is a lower position with its tag, at most a window back, and whose 64 bytes verify, is walked
 *     BACK to where the agreement starts (not past the segment start, not onto a lower sample -- every position has one owner);
 *     the candidate word there becomes (min(B2Z_CAP, bytes to the segment end), distance) unless stage F's candidate there is
 *     as long AND itself verifies 64 bytes (it is nearer, so cheaper).
 * Stage G prices the word like any other; chosen, it is extended by direct comparison to its true length (or the segment end). */
static void ldm_frame(const uint8_t *src, uint32_t n, const b2zo_enc_params *P, uint32_t *cand) {
    const uint32_t L = P->ldmLog, E = B2Z_LDM_EPOCHLOG(P->windowLog), nE = (uint32_t)(((uint64_t)n + (1u << E) - 1) >> E);
    const uint64_t W = 1ull << P->windowLog;
    const uint32_t tagMask = (1u << B2Z_LDM_TAGBITS) - 1;
    if (n < B2Z_LDM_MINMATCH) return;
    uint32_t *T = (uint32_t *)malloc(((size_t)nE << L) * 4);
    memset(T, 0xFF, ((size_t)nE << L) * 4);
    for (int pass = 0; pass < 2; pass++)
        for (uint32_t p = 0; p + B2Z_LDM_MINMATCH <= n; p++) {
            if (!b2z_ldm_sampled(rd64(src + p))) continue;
            const uint64_t key = b2z_ldm_key(rd64(src + p), rd64(src + p + 8), rd64(src + p + 16), rd64(src + p + 24));
            const uint32_t idx = (uint32_t)(key >> (64 - L)), tag = (uint32_t)(key >> (64 - L - B2Z_LDM_TAGBITS)) & tagMask;
            const uint32_t ep = p >> E;
            if (pass == 0) { uint32_t *t = T + ((size_t)ep << L) + idx; const uint32_t e = ((p - (ep << E)) << B2Z_LDM_TAGBITS) | tag; if (e < *t) *t = e; continue; }
            uint32_t d = 0;
            for (uint32_t back = 0; back <= 2 && back <= ep && !d; back++) {
                const uint32_t e = T[((size_t)(ep - back) << L) + idx];
                if (e == 0xFFFFFFFFu || (e & tagMask) != tag) continue;
                const uint32_t q = ((ep - back) << E) + (e >> B2Z_LDM_TAGBITS);
                if (q >= p || p - q >= W) continue;                              /* the first occurrence itself / beyond the window */
                if (count_match(src + q, src + p, B2Z_LDM_MINMATCH) >= B2Z_LDM_MINMATCH) d = p - q;
            }
            if (!d) continue;
            uint32_t s0 = p; const uint32_t segStart = p & ~(B2Z_SEG - 1);
            while (s0 > segStart && s0 > d && src[s0 - 1] == src[s0 - 1 - d] && !b2z_ldm_sampled(rd64(src + s0 - 1))) s0--;
            const uint32_t segEnd = ((p | (B2Z_SEG - 1)) + 1) < n ? ((p | (B2Z_SEG - 1)) + 1) : n;
            const uint32_t maxLen = segEnd - s0 > B2Z_CAP ? B2Z_CAP : segEnd - s0;
            if (maxLen < B2Z_DP_MINLEN) continue;
            const uint32_t c = cand[s0];
            if (c && B2Z_CAND_LEN(c) >= maxLen &&
                (maxLen < B2Z_CAP || count_match(src + s0 - B2Z_CAND_OFF(c), src + s0, B2Z_LDM_MINMATCH) >= B2Z_LDM_MINMATCH)) continue;
            cand[s0] = B2Z_CAND(maxLen, d);
        }
    free(T);
}

/* candidate words of one frame: stage F per region, then stage L */
void b2zo_zstd_candidates(const void *srcv, uint32_t n, const b2zo_enc_params *P, uint32_t *cand) {
    const uint8_t *src = (const uint8_t *)srcv;
    const uint32_t RL = P->regionLog && P->regionLog < P->frameLog ? P->regionLog : P->frameLog, R = 1u << RL;
    for (uint32_t r0 = 0; r0 < n || r0 == 0; r0 += R) {
        candidates_region(src + r0, n - r0 < R ? n - r0 : R, P, RL, cand + r0);
        if (n - r0 <= R) break;
    }
    if (P->ldmLog) ldm_frame(src, n, P, cand);
}

typedef struct { uint32_t rep[3]; } seg_rep_t;

/* Stage G, one frame: candidate words -> per 128 KiB block final sequences (B2Z_PACK_SEQ) and literal bytes.
 *
 * The role of the parse in ZSTD_compressBlock_doubleFast (greedy + repcode check) is played by a minimum-price path:
 * a block is cut into SEGMENTS of 4 KiB (one GPU lane each, a warp per block); inside a segment a backward dynamic
 * programme prices, at every position, the literal (its byte's cost in the block's sampled histogram) against the
 * position's candidate at its full length and at up to B2Z_DP_NTRUNC shorter lengths (B2Z_DP_MATCH + the offset's extra
 * bits; lengths up to B2Z_CAP have no extra bits).  The forward walk follows the choices; a chosen match of the full B2Z_CAP bytes is extended
 * by direct comparison to the segment end and the walk continues with the choice stored where the match ends.
 * Offsets become offBase with a repcode history that starts "unknown" at every segment (ZSTD_updateRep rules,
 * zstd_compress_internal.h:817-835), so lanes are independent; literal runs carry across segments.
 * A block of one repeated byte is emitted as the single sequence stage E turns into an RLE block. */
static void parse_frame(const uint8_t *src, uint32_t n, const uint32_t *cand,
                        uint64_t *seqs, uint32_t *nseq, uint8_t *lits, uint32_t *nlit) {
    static const zop_tables ZT = ZOP_TABLES_INIT;
    uint32_t *cost = (uint32_t *)malloc((B2Z_SEG + 1) * 4);
    uint8_t *choice = (uint8_t *)malloc(B2Z_SEG);
    const uint32_t nblocks = (n + ZF_BLOCK_MAX - 1) / ZF_BLOCK_MAX;
    for (uint32_t blk = 0; blk < nblocks; blk++) {
        const uint32_t b0 = blk * ZF_BLOCK_MAX, bn = n - b0 < ZF_BLOCK_MAX ? n - b0 : ZF_BLOCK_MAX;
        const uint8_t *bs = src + b0;
        uint64_t *out = seqs + (size_t)blk * B2Z_MAXSEQ;
        uint8_t *lit = lits + b0;
        uint32_t ns = 0, nl = 0;
        /* one repeated byte */
        { uint32_t i = 1; while (i < bn && bs[i] == bs[0]) i++;
          if (i == bn && bn > 1) { out[0] = B2Z_PACK_SEQ(1 + 3, 1, bn - 1); lit[0] = bs[0]; nseq[blk] = 1; nlit[blk] = 1; continue; } }
        /* literal prices from the sampled histogram */
        uint32_t hist[256] = { 0 }, tot = 0, lc[256];
        for (uint32_t i = 0; i < bn; i++) if (B2Z_DP_SAMPLED(i)) { hist[bs[i]]++; tot++; }
        for (uint32_t c = 0; c < 256; c++) {
            uint32_t v = hist[c] ? zop_cost(&ZT, hist[c], tot) : B2Z_DP_LIT_MAX;
            lc[c] = v < B2Z_DP_LIT_MIN ? B2Z_DP_LIT_MIN : (v > B2Z_DP_LIT_MAX ? B2Z_DP_LIT_MAX : v);
        }
        uint32_t prevEnd = 0;                                                   /* block-relative end of the last sequence */
        for (uint32_t s0 = 0; s0 < bn; s0 += B2Z_SEG) {
            const uint32_t s1 = bn - s0 < B2Z_SEG ? bn : s0 + B2Z_SEG, sn = s1 - s0;
            cost[sn] = 0;
            for (uint32_t i = sn; i-- > 0;) {
                const uint32_t c = cand[b0 + s0 + i];
                uint32_t best = lc[bs[s0 + i]] + cost[i + 1], ch = 0;
                if (c) {
                    const uint32_t len = B2Z_CAND_LEN(c), ob = 16 * zf_highbit32(B2Z_CAND_OFF(c) + 3) + B2Z_DP_MATCH;
                    for (uint32_t k = 0; k <= B2Z_DP_NTRUNC && len >= B2Z_DP_MINLEN + k; k++) {
                        const uint32_t l = len - k, pr = ob + cost[i + l];
                        if (pr < best) { best = pr; ch = l; }
                    }
                }
                cost[i] = best; choice[i] = (uint8_t)ch;
            }
            seg_rep_t R = { { 0, 0, 0 } };
            for (uint32_t i = 0; i < sn;) {
                uint32_t l = choice[i];
                if (!l) { lit[nl++] = bs[s0 + i]; i++; continue; }
                const uint32_t pos = s0 + i, off = B2Z_CAND_OFF(cand[b0 + pos]);
                if (l == B2Z_CAP) { const uint8_t *a = bs + pos, *q = a - off;             /* q may point into an earlier block of the frame */
                                    while (i + l < sn && a[l] == q[l]) l++; }
                const uint32_t ll = pos - prevEnd, ll0 = ll == 0;
                uint32_t code = 0, offBase;
                if (!ll0) { if (off == R.rep[0]) code = 1; else if (off == R.rep[1]) code = 2; else if (off == R.rep[2]) code = 3; }
                else { if (off == R.rep[1]) code = 1; else if (off == R.rep[2]) code = 2; else if (R.rep[0] > 1 && off == R.rep[0] - 1) code = 3; }
                if (code == 0) { offBase = off + 3; R.rep[2] = R.rep[1]; R.rep[1] = R.rep[0]; R.rep[0] = off; }
                else {
                    offBase = code;
                    const uint32_t idx = code - 1 + ll0;
                    if (idx != 0) { const uint32_t cur = idx == 3 ? R.rep[0] - 1 : R.rep[idx]; if (idx != 1) R.rep[2] = R.rep[1]; R.rep[1] = R.rep[0]; R.rep[0] = cur; }
                }
                out[ns++] = B2Z_PACK_SEQ(offBase, ll, l);
                prevEnd = pos + l; i += l;
            }
        }
        nseq[blk] = ns; nlit[blk] = nl;
    }
    free(cost); free(choice);
}

static void find_sequences_frame(const uint8_t *src, size_t n, const b2zo_enc_params *P,
                                 uint64_t *seqs, uint32_t *nseq, uint8_t *lits, uint32_t *nlit) {
    uint32_t *cand = (uint32_t *)malloc((n + 1) * 4);
    b2zo_zstd_candidates(src, (uint32_t)n, P, cand);
    parse_frame(src, (uint32_t)n, cand, seqs, nseq, lits, nlit);
    free(cand);
}

int64_t b2zo_zstd_find_sequences(const void *srcv, size_t srcSize, const b2zo_enc_params *P,
                                 uint64_t *seqs, uint32_t *nseq, uint8_t *lits, uint32_t *nlit) {
    const uint8_t *src = (const uint8_t *)srcv;
    size_t F = (size_t)1 << P->frameLog, blkBase = 0;
    for (size_t f0 = 0; f0 < srcSize; f0 += F) {
        size_t fn = srcSize - f0 < F ? srcSize - f0 : F;
        if (P->flags & B2Z_FLAG_ZSTD_OPT) b2zo_zstd_parse_frame(src + f0, (uint32_t)fn, P, NULL, seqs + blkBase * B2Z_MAXSEQ, nseq + blkBase, lits + f0, nlit + blkBase);
        else find_sequences_frame(src + f0, fn, P, seqs + blkBase * B2Z_MAXSEQ, nseq + blkBase, lits + f0, nlit + blkBase);
        blkBase += (fn + ZF_BLOCK_MAX - 1) / ZF_BLOCK_MAX;
    }
    return (int64_t)blkBase;
}

/* ======================================================================= stage E helpers */
typedef struct { uint8_t *p; uint64_t acc; uint32_t nb; } bitw_t;       /* LSB-first writer */
static inline void bw_init(bitw_t *b, uint8_t *p) { b->p = p; b->acc = 0; b->nb = 0; }
static inline void bw_add(bitw_t *b, uint32_t v, uint32_t n) {           /* n <= 32 */
    b->acc |= (uint64_t)(v & (n == 32 ? 0xFFFFFFFFu : ((1u << n) - 1))) << b->nb; b->nb += n;
    while (b->nb >= 8) { *b->p++ = (uint8_t)b->acc; b->acc >>= 8; b->nb -= 8; }
}
static inline uint8_t *bw_close(bitw_t *b) {                             /* end mark + pad */
    bw_add(b, 1, 1);
    if (b->nb) { *b->p++ = (uint8_t)b->acc; b->acc = 0; b->nb = 0; }
    return b->p;
}

/* ---- FSE encoding tables -------------------------------------------------------------- */
typedef struct { int32_t deltaFindState; uint32_t deltaNbBits; } fse_symtt;
typedef struct { uint16_t state[512]; fse_symtt tt[64]; uint32_t log; } fse_ctable;

static void fse_build_ctable(fse_ctable *ct, const int16_t *norm, uint32_t maxSym, uint32_t log) {
    uint32_t size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    uint8_t spread[512]; uint32_t cumul[65], high = size - 1;
    cumul[0] = 0;
    for (uint32_t s = 0; s <= maxSym; s++) {
        if (norm[s] == -1) { cumul[s + 1] = cumul[s] + 1; spread[high--] = (uint8_t)s; }
        else cumul[s + 1] = cumul[s] + (uint32_t)norm[s];
    }
    uint32_t pos = 0;
    for (uint32_t s = 0; s <= maxSym; s++)
        for (int i = 0; i < norm[s]; i++) { spread[pos] = (uint8_t)s; pos = (pos + step) & mask; while (pos > high) pos = (pos + step) & mask; }
    for (uint32_t u = 0; u < size; u++) { uint32_t s = spread[u]; ct->state[cumul[s]++] = (uint16_t)(size + u); }
    uint32_t total = 0;
    for (uint32_t s = 0; s <= maxSym; s++) {
        int n = norm[s];
        if (n == 0) { ct->tt[s].deltaNbBits = ((log + 1) << 16) - size; ct->tt[s].deltaFindState = 0; }
        else if (n == 1 || n == -1) { ct->tt[s].deltaNbBits = (log << 16) - size; ct->tt[s].deltaFindState = (int32_t)total - 1; total++; }
        else {
            uint32_t maxBitsOut = log - zf_highbit32((uint32_t)n - 1), minStatePlus = (uint32_t)n << maxBitsOut;
            ct->tt[s].deltaNbBits = (maxBitsOut << 16) - minStatePlus;
            ct->tt[s].deltaFindState = (int32_t)total - n; total += (uint32_t)n;
        }
    }
    ct->log = log;
}
static inline uint32_t fse_init_state(const fse_ctable *ct, uint32_t sym) {
    uint32_t nb = (ct->tt[sym].deltaNbBits + (1u << 15)) >> 16;
    uint32_t v = (nb << 16) - ct->tt[sym].deltaNbBits;
    return ct->state[(v >> nb) + ct->tt[sym].deltaFindState];
}
static inline uint32_t fse_encode(const fse_ctable *ct, uint32_t *state, uint32_t sym, uint32_t *nbOut) {
    uint32_t nb = (*state + ct->tt[sym].deltaNbBits) >> 16, bits = *state & ((1u << nb) - 1);
    *state = ct->state[(*state >> nb) + ct->tt[sym].deltaFindState];
    *nbOut = nb; return bits;
}

/* ---- normalisation (own scheme; any valid normalisation is format-legal) ------------------
 * norm[s] = max(1, round(count*2^log/total)) for present symbols, then the rounding error is
 * settled on the largest entries.  No "-1" (low-probability) entries are produced. */
static void fse_normalize(int16_t *norm, uint32_t log, const uint32_t *count, uint32_t total, uint32_t maxSym) {
    uint32_t size = 1u << log; int32_t sum = 0;
    for (uint32_t s = 0; s <= maxSym; s++) {
        if (!count[s]) { norm[s] = 0; continue; }
        uint64_t p = ((uint64_t)count[s] * size * 2 + total) / (2ull * total);
        if (p < 1) p = 1;
        norm[s] = (int16_t)p; sum += (int32_t)p;
    }
    int32_t delta = (int32_t)size - sum;
    while (delta != 0) {                                    /* settle on the currently largest entry */
        uint32_t big = 0;
        for (uint32_t s = 1; s <= maxSym; s++) if (norm[s] > norm[big]) big = s;
        if (delta > 0) { norm[big] = (int16_t)(norm[big] + delta); delta = 0; }
        else {
            int32_t take = norm[big] - 1 < -delta ? norm[big] - 1 : -delta;
            if (take > (norm[big] >> 1) && norm[big] > 2) take = norm[big] >> 1;   /* spread large deficits */
            norm[big] = (int16_t)(norm[big] - take); delta += take;
        }
    }
}

/* Serialise normalised counts (fse_compress.c:233-345 semantics). Returns bytes written. */
static size_t fse_write_ncount(uint8_t *dst, const int16_t *norm, uint32_t maxSym, uint32_t log) {
    bitw_t b; bw_init(&b, dst);
    bw_add(&b, log - 5, 4);
    int32_t remaining = (int32_t)(1u << log);
    uint32_t s = 0;
    while (remaining > 0 && s <= maxSym) {
        int nb = (int)zf_highbit32((uint32_t)remaining + 1) + 1;
        uint32_t T = 1u << (nb - 1), max = 2 * T - 1 - ((uint32_t)remaining + 1);
        int32_t proba = norm[s++];
        uint32_t count = (uint32_t)(proba + 1);
        remaining -= proba < 0 ? 1 : proba;
        if (count < max) bw_add(&b, count, (uint32_t)nb - 1);
        else if (count < T) bw_add(&b, count, (uint32_t)nb);
        else bw_add(&b, count + max, (uint32_t)nb);
        if (proba == 0) {                                   /* run of zeros: 2-bit repeat counts */
            for (;;) {
                uint32_t run = 0;
                while (run < 3 && s <= maxSym && norm[s] == 0) { run++; s++; }
                bw_add(&b, run, 2);
                if (run < 3) break;
            }
        }
    }
    if (b.nb) { *b.p++ = (uint8_t)b.acc; }
    return (size_t)(b.p - dst);
}

/* ---- fixed-point costs ------------------------------------------------------------------ */
/* log2(x) * 256 for x >= 1, integer only (8 fractional bits from a 32-entry mantissa table) */
static uint32_t log2_fx8(uint32_t x) {
    static const uint8_t frac[32] = { 0, 11, 22, 33, 43, 53, 63, 72, 82, 91, 100, 108, 116, 125, 132, 140,
                                      148, 155, 162, 169, 176, 182, 189, 195, 201, 207, 213, 219, 225, 230, 236, 241 };
    uint32_t hb = zf_highbit32(x);
    uint32_t m = hb >= 5 ? (x >> (hb - 5)) & 31 : (x << (5 - hb)) & 31;
    return (hb << 8) + frac[m];
}
/* cost in 1/256 bit of coding `count` with table (norm, log) */
static uint64_t fse_cost_fx8(const uint32_t *count, const int16_t *norm, uint32_t maxSym, uint32_t log) {
    uint64_t c = 0;
    for (uint32_t s = 0; s <= maxSym; s++) {
        if (!count[s]) continue;
        if (norm[s] == 0) return ~0ull;                     /* symbol not representable */
        uint32_t n = norm[s] < 0 ? 1u : (uint32_t)norm[s];
        c += (uint64_t)count[s] * ((log << 8) - log2_fx8(n));
    }
    return c;
}

/* ======================================================================= Huffman */
typedef struct { uint16_t code[256]; uint8_t len[256]; uint32_t maxBits; uint32_t maxSym; } huf_ctable;

/* Code lengths by the textbook two-queue construction on (count, symbol)-sorted leaves; if the
 * tree is deeper than 11 the counts are halved (floor at 1) and the tree rebuilt -- always a
 * complete prefix code, hence representable as zstd weights. */
static void huf_build(huf_ctable *h, const uint32_t *count0) {
    uint32_t count[256];
    uint32_t order[256], n;
    for (uint32_t k = 0;; k++) {                            /* k = number of halvings: ceil(count / 2^k) */
        for (uint32_t s = 0; s < 256; s++) count[s] = count0[s] ? (count0[s] + (1u << k) - 1) >> k : 0;
        n = 0;
        for (uint32_t s = 0; s < 256; s++) if (count[s]) order[n++] = s;
        /* stable sort by count ascending (symbols already ascending) */
        for (uint32_t i = 1; i < n; i++) { uint32_t s = order[i]; int j = (int)i - 1; while (j >= 0 && count[order[j]] > count[s]) { order[j + 1] = order[j]; j--; } order[j + 1] = s; }
        uint32_t w[512]; int parent[512];
        for (uint32_t i = 0; i < n; i++) w[i] = count[order[i]];
        uint32_t li = 0, ii = n, ie = n;                    /* leaf head, internal head, internal end */
        while ((n - li) + (ie - ii) > 1) {
            uint32_t a, b;
            if (li < n && (ii >= ie || w[li] <= w[ii])) a = li++; else a = ii++;
            if (li < n && (ii >= ie || w[li] <= w[ii])) b = li++; else b = ii++;
            w[ie] = w[a] + w[b]; parent[a] = (int)ie; parent[b] = (int)ie; ie++;
        }
        uint32_t depth[512], maxd = 0; depth[ie - 1] = 0;
        for (int i = (int)ie - 2; i >= 0; i--) depth[i] = depth[parent[i]] + 1;
        for (uint32_t i = 0; i < n; i++) if (depth[i] > maxd) maxd = depth[i];
        if (maxd <= ZF_HUF_MAXBITS) {
            memset(h->len, 0, 256);
            for (uint32_t i = 0; i < n; i++) h->len[order[i]] = (uint8_t)depth[i];
            h->maxBits = maxd; h->maxSym = order[0];
            for (uint32_t s = 0; s < 256; s++) if (count[s]) h->maxSym = s;
            break;
        }
    }
    /* canonical values in zstd order: weight w = maxBits+1-len; cells filled by ascending weight,
       symbols ascending inside a weight; value = firstCell >> (w-1) */
    uint32_t rank[ZF_HUF_MAXBITS + 2] = { 0 }, start[ZF_HUF_MAXBITS + 2], pos = 0;
    for (uint32_t s = 0; s < 256; s++) if (h->len[s]) rank[h->maxBits + 1 - h->len[s]]++;
    for (uint32_t r = 1; r <= h->maxBits; r++) { start[r] = pos; pos += rank[r] << (r - 1); }
    for (uint32_t s = 0; s < 256; s++) {
        if (!h->len[s]) { h->code[s] = 0; continue; }
        uint32_t r = h->maxBits + 1 - h->len[s];
        h->code[s] = (uint16_t)(start[r] >> (r - 1)); start[r] += 1u << (r - 1);
    }
}

/* Tree description: FSE-compressed weights when that is smaller than raw nibbles.
 * Returns bytes written, 0 if not representable (caller stores literals raw). */
static size_t huf_write_table(uint8_t *dst, const huf_ctable *h) {
    uint8_t w[256]; uint32_t nw = h->maxSym;                /* last weight is implicit */
    for (uint32_t s = 0; s < nw; s++) w[s] = h->len[s] ? (uint8_t)(h->maxBits + 1 - h->len[s]) : 0;
    size_t fseSize = 0; uint8_t tmp[160];
    if (nw > 1) {
        uint32_t cnt[16] = { 0 }, maxW = 0, maxCnt = 0;
        for (uint32_t i = 0; i < nw; i++) { cnt[w[i]]++; if (w[i] > maxW) maxW = w[i]; }
        for (uint32_t i = 0; i <= maxW; i++) if (cnt[i] > maxCnt) maxCnt = cnt[i];
        if (maxCnt != nw && maxCnt > 1) {
            uint32_t log = 6;                               /* weights table log: <= 6 */
            uint32_t minBits = zf_highbit32(nw) + 1, symBits = zf_highbit32(maxW + 1) + 2;
            uint32_t lo = minBits < symBits ? minBits : symBits;
            uint32_t want = zf_highbit32(nw - 1) >= 2 ? zf_highbit32(nw - 1) - 2 : 0;
            if (want < log) log = want;
            if (log < lo) log = lo;
            if (log < 5) log = 5;
            if (log > 6) log = 6;
            int16_t norm[16]; fse_normalize(norm, log, cnt, nw, maxW);
            size_t hs = fse_write_ncount(tmp, norm, maxW, log);
            fse_ctable ct; fse_build_ctable(&ct, norm, maxW, log);
            bitw_t b; bw_init(&b, tmp + hs);
            /* two interleaved states, symbols walked last -> first (fse_compress.c:558-622 order) */
            uint32_t i = nw, s1, s2, nb, bits;
            if (nw & 1) { s1 = fse_init_state(&ct, w[--i]); s2 = fse_init_state(&ct, w[--i]);
                          bits = fse_encode(&ct, &s1, w[--i], &nb); bw_add(&b, bits, nb); }
            else { s2 = fse_init_state(&ct, w[--i]); s1 = fse_init_state(&ct, w[--i]); }
            while (i > 0) {
                bits = fse_encode(&ct, &s2, w[--i], &nb); bw_add(&b, bits, nb);
                bits = fse_encode(&ct, &s1, w[--i], &nb); bw_add(&b, bits, nb);
            }
            bw_add(&b, s2, log); bw_add(&b, s1, log);
            fseSize = (size_t)(bw_close(&b) - tmp);
        }
    }
    size_t rawSize = (nw + 1) / 2;
    if (fseSize && fseSize < 128 && (fseSize < rawSize || nw > 128)) {
        dst[0] = (uint8_t)fseSize; memcpy(dst + 1, tmp, fseSize); return 1 + fseSize;
    }
    if (nw > 128 || nw == 0) return 0;
    dst[0] = (uint8_t)(127 + nw);
    for (uint32_t i = 0; i < nw; i += 2) dst[1 + i / 2] = (uint8_t)((w[i] << 4) | (i + 1 < nw ? w[i + 1] : 0));
    return 1 + rawSize;
}

static size_t huf_encode_stream(uint8_t *dst, const uint8_t *lit, size_t n, const huf_ctable *h) {
    bitw_t b; bw_init(&b, dst);
    for (size_t i = n; i-- > 0;) bw_add(&b, h->code[lit[i]], h->len[lit[i]]);
    return (size_t)(bw_close(&b) - dst);
}

/* Literals section. Returns bytes written. */
static size_t write_literals(uint8_t *dst, const uint8_t *lit, size_t n) {
    uint32_t count[256] = { 0 }, ns = 0;
    for (size_t i = 0; i < n; i++) count[lit[i]]++;
    for (uint32_t s = 0; s < 256; s++) ns += count[s] != 0;
    size_t rawHdr = n < 32 ? 1 : (n < 4096 ? 2 : 3);
    if (n >= B2Z_LIT_RLE_MIN && ns == 1) {                  /* RLE literals */
        if (rawHdr == 1) dst[0] = (uint8_t)(1 | (n << 3));
        else if (rawHdr == 2) wr16(dst, (uint32_t)(1 | (1 << 2) | (n << 4)));
        else wr24(dst, (uint32_t)(1 | (3 << 2) | (n << 4)));
        dst[rawHdr] = lit[0]; return rawHdr + 1;
    }
    if (n >= B2Z_LIT_HUF_MIN && ns >= 2) {
        huf_ctable h; huf_build(&h, count);
        uint8_t *tmp = (uint8_t *)malloc(n + n / 2 + 512);
        size_t ts = huf_write_table(tmp, &h);
        if (ts) {
            int four = n >= 256;
            size_t lh = n < 1024 ? 3 : (n < 16384 ? 4 : 5);
            uint64_t T = 0;                                 /* exact payload bits; decision on the byte bound */
            for (uint32_t sy = 0; sy < 256; sy++) T += (uint64_t)count[sy] * h.len[sy];
            size_t est = ts + (four ? 6 : 0) + (size_t)((T + 7) / 8) + (four ? 4 : 1);
            if (lh + est < rawHdr + n) {
                uint8_t *p = tmp + ts; size_t body;
                if (!four) body = huf_encode_stream(p, lit, n, &h);
                else {
                    size_t seg = (n + 3) / 4; uint8_t *q = p + 6; size_t s;
                    s = huf_encode_stream(q, lit, seg, &h); wr16(p, (uint32_t)s); q += s;
                    s = huf_encode_stream(q, lit + seg, seg, &h); wr16(p + 2, (uint32_t)s); q += s;
                    s = huf_encode_stream(q, lit + 2 * seg, seg, &h); wr16(p + 4, (uint32_t)s); q += s;
                    s = huf_encode_stream(q, lit + 3 * seg, n - 3 * seg, &h); q += s;
                    body = (size_t)(q - p);
                }
                size_t csize = ts + body;
                uint32_t sf = !four ? 0 : (lh == 3 ? 1 : (lh == 4 ? 2 : 3));
                if (lh == 3) wr24(dst, (uint32_t)(2 | (sf << 2) | (n << 4) | (csize << 14)));
                else if (lh == 4) wr32(dst, (uint32_t)(2 | (sf << 2) | (n << 4) | (csize << 18)));
                else { uint64_t v = 2 | (sf << 2) | ((uint64_t)n << 4) | ((uint64_t)csize << 22); wr32(dst, (uint32_t)v); dst[4] = (uint8_t)(v >> 32); }
                memcpy(dst + lh, tmp, csize); free(tmp);
                return lh + csize;
            }
        }
        free(tmp);
    }
    /* raw literals */
    if (rawHdr == 1) dst[0] = (uint8_t)(n << 3);
    else if (rawHdr == 2) wr16(dst, (uint32_t)((1 << 2) | (n << 4)));
    else wr24(dst, (uint32_t)((3 << 2) | (n << 4)));
    memcpy(dst + rawHdr, lit, n);
    return rawHdr + n;
}

/* ======================================================================= sequences */
typedef struct { uint32_t ll, ml, offBase; } fseq_t;

/* choose table mode for one symbol type and serialise its description */
typedef struct { fse_ctable ct; uint32_t mode; } seq_table_choice;
static size_t choose_seq_table(seq_table_choice *ch, uint8_t *dst, const uint8_t *codes, uint32_t nbSeq,
                               uint32_t maxSymAll, uint32_t maxLog, const int16_t *defNorm, uint32_t defMaxSym, uint32_t defLog) {
    uint32_t count[64] = { 0 }, maxSym = 0, present = 0, big = 0;
    for (uint32_t i = 0; i < nbSeq; i++) count[codes[i]]++;
    for (uint32_t s = 0; s <= maxSymAll; s++) if (count[s]) { maxSym = s; present++; if (count[s] > big) big = count[s]; }
    if (big == nbSeq && !(nbSeq <= 2 && maxSym <= defMaxSym)) {   /* RLE: single zero-bit state */
        memset(&ch->ct, 0, sizeof(ch->ct));
        ch->mode = 1; dst[0] = (uint8_t)maxSym; return 1;
    }
    uint64_t costDef = maxSym <= defMaxSym ? fse_cost_fx8(count, defNorm, maxSym, defLog) : ~0ull;
    /* compressed */
    uint32_t log = zf_highbit32(nbSeq > 1 ? nbSeq - 1 : 1) >= 2 ? zf_highbit32(nbSeq > 1 ? nbSeq - 1 : 1) - 2 : 0;
    uint32_t minA = zf_highbit32(nbSeq) + 1, minB = zf_highbit32(maxSym ? maxSym : 1) + 2, lo = minA < minB ? minA : minB;
    if (log > maxLog) log = maxLog;
    if (log < lo) log = lo;
    if (log < 5) log = 5;
    if (log > maxLog) log = maxLog;
    while ((1u << log) < present) log++;
    int16_t norm[64]; uint8_t hdr[64];
    fse_normalize(norm, log, count, nbSeq, maxSym);
    size_t hs = fse_write_ncount(hdr, norm, maxSym, log);
    uint64_t costFse = fse_cost_fx8(count, norm, maxSym, log) + ((uint64_t)hs << 11);
    if (costDef <= costFse || big == nbSeq) {
        fse_build_ctable(&ch->ct, defNorm, defMaxSym, defLog); ch->mode = 0; return 0;
    }
    fse_build_ctable(&ch->ct, norm, maxSym, log); ch->mode = 2; memcpy(dst, hdr, hs); return hs;
}

/* returns section size, or (size_t)-1 when litSize + the section's size upper bound exceeds B2Z_BODY_CAP */
static size_t write_sequences(uint8_t *dst, const fseq_t *seq, uint32_t nbSeq, size_t litSize) {
    uint8_t *op = dst;
    if (nbSeq < 128) *op++ = (uint8_t)nbSeq;
    else if (nbSeq < 0x7F00) { *op++ = (uint8_t)((nbSeq >> 8) + 128); *op++ = (uint8_t)nbSeq; }
    else { *op++ = 255; wr16(op, nbSeq - 0x7F00); op += 2; }
    if (nbSeq == 0) return (size_t)(op - dst);
    uint8_t *llc = (uint8_t *)malloc(3 * (size_t)nbSeq), *ofc = llc + nbSeq, *mlc = ofc + nbSeq;
    for (uint32_t i = 0; i < nbSeq; i++) {
        llc[i] = (uint8_t)zf_ll_code(seq[i].ll); mlc[i] = (uint8_t)zf_ml_code(seq[i].ml - 3); ofc[i] = (uint8_t)zf_highbit32(seq[i].offBase);
    }
    uint8_t *modes = op++;
    seq_table_choice L, O, M;
    op += choose_seq_table(&L, op, llc, nbSeq, ZF_MAXLL, ZF_LL_FSELOG, ZF_LL_defaultNorm, 35, ZF_LL_DEFLOG);
    op += choose_seq_table(&O, op, ofc, nbSeq, ZF_MAXOFF, ZF_OF_FSELOG, ZF_OF_defaultNorm, 28, ZF_OF_DEFLOG);
    op += choose_seq_table(&M, op, mlc, nbSeq, ZF_MAXML, ZF_ML_FSELOG, ZF_ML_defaultNorm, 52, ZF_ML_DEFLOG);
    *modes = (uint8_t)((L.mode << 6) | (O.mode << 4) | (M.mode << 2));
    {
        uint64_t upper = (uint64_t)nbSeq * (L.ct.log + O.ct.log + M.ct.log) + 1;
        for (uint32_t k = 0; k < nbSeq; k++) upper += ZF_LL_bits[llc[k]] + ZF_ML_bits[mlc[k]] + ofc[k];
        if (litSize + (size_t)(op - dst) + (size_t)((upper + 7) / 8) > B2Z_BODY_CAP) { free(llc); return (size_t)-1; }
    }
    bitw_t b; bw_init(&b, op);
    uint32_t i = nbSeq - 1, nb, bits;
    uint32_t sM = fse_init_state(&M.ct, mlc[i]), sO = fse_init_state(&O.ct, ofc[i]), sL = fse_init_state(&L.ct, llc[i]);
    bw_add(&b, seq[i].ll - ZF_LL_base[llc[i]], ZF_LL_bits[llc[i]]);
    bw_add(&b, seq[i].ml - ZF_ML_base[mlc[i]], ZF_ML_bits[mlc[i]]);
    bw_add(&b, seq[i].offBase - (1u << ofc[i]), ofc[i]);
    while (i-- > 0) {
        bits = fse_encode(&O.ct, &sO, ofc[i], &nb); bw_add(&b, bits, nb);
        bits = fse_encode(&M.ct, &sM, mlc[i], &nb); bw_add(&b, bits, nb);
        bits = fse_encode(&L.ct, &sL, llc[i], &nb); bw_add(&b, bits, nb);
        bw_add(&b, seq[i].ll - ZF_LL_base[llc[i]], ZF_LL_bits[llc[i]]);
        bw_add(&b, seq[i].ml - ZF_ML_base[mlc[i]], ZF_ML_bits[mlc[i]]);
        bw_add(&b, seq[i].offBase - (1u << ofc[i]), ofc[i]);
    }
    bw_add(&b, sM, M.ct.log); bw_add(&b, sO, O.ct.log); bw_add(&b, sL, L.ct.log);
    op = bw_close(&b);
    free(llc);
    return (size_t)(op - dst);
}

/* One block: returns bytes written including the 3-byte header. */
static size_t compress_block(uint8_t *dst, const uint8_t *frame, size_t blkStart, size_t blkSize, int last,
                             const uint64_t *packed, uint32_t nbSeq, const uint8_t *lits, uint32_t nlit) {
    fseq_t *seq = (fseq_t *)malloc(sizeof(fseq_t) * (nbSeq + 1));
    for (uint32_t i = 0; i < nbSeq; i++) { seq[i].offBase = B2Z_SEQ_OFFBASE(packed[i]); seq[i].ll = B2Z_SEQ_LL(packed[i]); seq[i].ml = B2Z_SEQ_ML(packed[i]); }
    const uint8_t *src = frame + blkStart;
    size_t out;
    if (blkSize > 1 && nbSeq == 1 && nlit == 1 && seq[0].ll == 1 && seq[0].ml == blkSize - 1 && seq[0].offBase == 1 + 3) {
        wr24(dst, (uint32_t)(last | (1 << 1) | (blkSize << 3))); dst[3] = src[0]; out = 4;   /* RLE block */
    } else {
        uint8_t *body = (uint8_t *)malloc(B2Z_BODY_CAP + 1024);
        size_t ls = write_literals(body, lits, nlit);
        size_t ss = write_sequences(body + ls, seq, nbSeq, ls);
        if (ss != (size_t)-1 && ls + ss < blkSize) { wr24(dst, (uint32_t)(last | (2 << 1) | ((ls + ss) << 3))); memcpy(dst + 3, body, ls + ss); out = 3 + ls + ss; }
        else { wr24(dst, (uint32_t)(last | (blkSize << 3))); memcpy(dst + 3, src, blkSize); out = 3 + blkSize; }
        free(body);
    }
    free(seq);
    return out;
}

static size_t write_frame_header(uint8_t *dst, size_t n, const b2zo_enc_params *P) {
    wr32(dst, ZF_MAGIC);
    if (n == 0) { dst[4] = (uint8_t)(0x20 | ((P->flags & 2) ? 4 : 0)); dst[5] = 0; return 6; }     /* single segment, FCS = 0 */
    uint32_t wl = 10; while (((size_t)1 << wl) < n && wl < P->windowLog) wl++;
    dst[4] = (uint8_t)(0x80 | ((P->flags & 2) ? 4 : 0));     /* 4-byte FCS, window descriptor present */
    dst[5] = (uint8_t)((wl - 10) << 3);
    wr32(dst + 6, (uint32_t)n);
    return 10;
}

int64_t b2zo_zstd_compress(void *dstv, size_t dstCap, const void *srcv, size_t srcSize, const b2zo_enc_params *P) {
    const uint8_t *src = (const uint8_t *)srcv; uint8_t *dst = (uint8_t *)dstv, *op = dst;
    if (dstCap < b2zo_zstd_compress_bound(srcSize, P)) return -2;
    size_t F = (size_t)1 << P->frameLog;
    size_t nblkMax = (F + ZF_BLOCK_MAX - 1) / ZF_BLOCK_MAX;
    uint64_t *seqs = (uint64_t *)malloc(sizeof(uint64_t) * B2Z_MAXSEQ * nblkMax);
    uint32_t *nseq = (uint32_t *)malloc(4 * nblkMax * 2), *nlit = nseq + nblkMax;
    uint8_t *lits = (uint8_t *)malloc(F);
    size_t f0 = 0;
    do {
        size_t fn = srcSize - f0 < F ? srcSize - f0 : F;
        const uint8_t *frame = src + f0;
        uint8_t *hint = NULL;
        if (P->flags & 1) { wr32(op, ZF_MAGIC_SKIP); wr32(op + 4, 4); hint = op + 8; op += 12; }
        uint8_t *fstart = op;
        op += write_frame_header(op, fn, P);
        if (fn == 0) { wr24(op, 1); op += 3; }
        else {
            if (P->flags & B2Z_FLAG_ZSTD_OPT) b2zo_zstd_parse_frame(frame, (uint32_t)fn, P, NULL, seqs, nseq, lits, nlit);
            else find_sequences_frame(frame, fn, P, seqs, nseq, lits, nlit);
            size_t nblk = (fn + ZF_BLOCK_MAX - 1) / ZF_BLOCK_MAX;
            for (size_t b = 0; b < nblk; b++) {
                size_t bs = b * ZF_BLOCK_MAX, bn = fn - bs < ZF_BLOCK_MAX ? fn - bs : ZF_BLOCK_MAX;
                op += compress_block(op, frame, bs, bn, b + 1 == nblk, seqs + b * B2Z_MAXSEQ, nseq[b], lits + bs, nlit[b]);
            }
        }
        if (P->flags & 2) { wr32(op, (uint32_t)b2zo_xxh64(frame, fn, 0)); op += 4; }
        if (hint) wr32(hint, (uint32_t)(op - fstart));
        f0 += fn;
    } while (f0 < srcSize);
    free(lits); free(nseq); free(seqs);
    return (int64_t)(op - dst);
}
