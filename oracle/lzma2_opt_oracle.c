/* lzma2_opt_oracle.c -- sequential statement of the price-based parse of the GPU LZMA2 encoder (method 21, flag B2Z_FLAG_LZ2_OPT).
 *
 * TEST INFRASTRUCTURE ONLY (see oracle.h).  States what csrc/lzma2_parse.cu computes:
 *
 *   stage C  candidates: for every position p of a frame and each of LZP_NCAND direct-mapped tables (keys of 3, 4, 6, 8 bytes),
 *            the NEAREST q < p whose key falls into the same table entry -- a pure function of the frame's bytes (the "last
 *            writer" of a table that every position updates, so any order of evaluation gives the same answer) -- with the
 *            common-prefix length of q and p.  Role in the reference: the match finders that hand the optimal parsers all
 *            (length, nearest distance) pairs -- LzFind.c:1219 Bt4_MatchFinder_GetMatches, fast-lzma2/radix_get.h:84 RMF_getMatch.
 *   stage P  parse: a forward dynamic programme over windows of at most LZP_WIN positions; node i holds the cheapest known way
 *            to have coded the window's first i bytes together with the coder state that way leaves (state, rep0-3); edges are
 *            literal / rep0-3 / match packets priced from the adaptive model as it stands at the window start; a window ends
 *            where all paths meet, at LZP_WIN nodes, or at a match of >= LZP_NICE bytes, which is taken at once; the chosen
 *            packets then update the model exactly as stage R will.  Role in the reference: LzmaEnc.c:1225 GetOptimum,
 *            fast-lzma2/lzma2_enc.c:949 LZMA_optimalParse (same idea; this formulation, its windows and its prices are ours).
 *   The packets leave as per-block sequences (literal run, match length, distance) in the layout stage R already consumes.
 */
#include <stdlib.h>
#include <string.h>
#include "oracle.h"
#include "b2z_params.h"
#include "b2z_lzma_model.h"

static const uint8_t PT[128] = { LZM_PRICE_LIST };

static uint32_t mlen(const uint8_t *b, uint32_t q, uint32_t p, uint32_t maxLen) { uint32_t l = 0; while (l < maxLen && b[q + l] == b[p + l]) l++; return l; }

/* ---------------------------------------------------------------------------------------------------------- stage C */
void b2zo_lzma2_candidates(const void *basev, uint32_t n, uint32_t frameLog, uint32_t *cand /* [n * LZP_NCAND] */) {
    const uint8_t *b = (const uint8_t *)basev;
    uint32_t *T[LZP_NCAND], lg[LZP_NCAND], kb[LZP_NCAND];
    for (uint32_t t = 0; t < LZP_NCAND; t++) { kb[t] = lzp_key_bytes(t); lg[t] = lzp_table_log(t, frameLog); T[t] = (uint32_t *)calloc((size_t)1 << lg[t], 4); }
    for (uint32_t p = 0; p < n; p++) {
        uint64_t v = 0; memcpy(&v, b + p, n - p < 8 ? n - p : 8);
        const uint32_t maxLen = n - p < B2Z_LZ2_MAXLEN ? n - p : B2Z_LZ2_MAXLEN;
        for (uint32_t t = 0; t < LZP_NCAND; t++) {
            uint32_t c = 0;
            if (p + kb[t] <= n) {
                uint32_t *e = T[t] + lzp_table_index(v, kb[t], lg[t]);
                const uint32_t q1 = *e;
                *e = p + 1;
                if (q1) {
                    const uint32_t l = mlen(b, q1 - 1, p, maxLen);
                    if (l >= 2) c = LZP_PACK_CAND(p - q1, l < LZP_CAND_LENCAP ? l : LZP_CAND_LENCAP);
                }
            }
            cand[(size_t)p * LZP_NCAND + t] = c;
        }
    }
    for (uint32_t t = 0; t < LZP_NCAND; t++) free(T[t]);
}

/* ---------------------------------------------------------------------------------------------------------- stage P */
enum { K_LIT = 0, K_REP = 1, K_MATCH = 2 };
typedef struct { uint32_t cost, from, kind, len, dist /* K_REP: rep index, K_MATCH: distance - 1 */; lzm_ctx x; } node_t;

typedef struct { uint64_t *seqs; uint32_t *nseq; uint32_t prevEnd; } sink_t;     /* block-indexed arrays of the frame */
static void sink_match(sink_t *s, uint32_t pos, uint32_t len, uint32_t dist) {
    const uint32_t b = pos >> 17, bs = b << 17;
    if (s->nseq[b] >= B2Z_MAXSEQ) return;                        /* block's array full: the bytes stay literals for stage R */
    const uint32_t from = s->prevEnd > bs ? s->prevEnd : bs;     /* literal runs are cut at block starts (stage R codes a block's tail itself) */
    s->seqs[(size_t)b * B2Z_MAXSEQ + s->nseq[b]++] = B2Z_PACK_SEQ(dist + 1u + 3u, pos - from, len);
    s->prevEnd = pos + len;
}
static void commit_literal(uint16_t *probs, lzm_ctx *x, const uint8_t *base, uint32_t p) {
    lzm_commit_literal(probs, x, p, p ? base[p - 1] : 0u, base[p], x->state >= 7u ? base[p - x->rep[0] - 1u] : 0u);
}

static void parse_slice(const uint8_t *base, uint32_t s0, uint32_t s1, const uint32_t *cand, uint16_t *probs, sink_t *sink, lzm_ctx *xOut) {
    node_t nd[LZP_WIN + 1];
    uint32_t path[LZP_WIN + 1];
    lzm_ctx x; x.state = 0; x.rep[0] = x.rep[1] = x.rep[2] = x.rep[3] = 0;
    for (uint32_t k = 0; k < LZM_NPROBS; k++) probs[k] = 1024;
    uint32_t pos = s0;
    while (pos < s1) {
        const uint32_t W = (s1 - pos) < LZP_WIN ? (s1 - pos) : LZP_WIN;
        nd[0].cost = 0; nd[0].x = x;
        for (uint32_t j = 1; j <= W; j++) nd[j].cost = 0xFFFFFFFFu;
        uint32_t end = 0, i = 0, longLen = 0, longDist = 0;
        for (;;) {
            if (i) {                                             /* node i is final: the coder state its best arrival leaves */
                node_t *y = &nd[i]; const node_t *f = &nd[y->from];
                y->x = f->x;
                if (y->kind == K_LIT) y->x.state = lzm_state_lit(f->x.state);
                else if (y->kind == K_REP) {
                    const uint32_t r = y->dist, d = f->x.rep[r];
                    for (uint32_t k = r; k > 0; k--) y->x.rep[k] = f->x.rep[k - 1];
                    y->x.rep[0] = d; y->x.state = lzm_state_rep(f->x.state);
                } else { y->x.rep[3] = f->x.rep[2]; y->x.rep[2] = f->x.rep[1]; y->x.rep[1] = f->x.rep[0]; y->x.rep[0] = y->dist; y->x.state = lzm_state_match(f->x.state); }
            }
            if (i == W || (i && i == end)) break;
            const uint32_t p = pos + i, st = nd[i].x.state, ps = p & LZM_PBM;
            const uint32_t *rep = nd[i].x.rep;
            const uint32_t maxLen = (s1 - p) < B2Z_LZ2_MAXLEN ? (s1 - p) : B2Z_LZ2_MAXLEN;
            const uint32_t *c = cand + (size_t)p * LZP_NCAND;
            uint32_t rl[4], cl[LZP_NCAND], cd[LZP_NCAND];
            for (uint32_t r = 0; r < 4; r++) {                   /* a rep equal to an earlier one is the earlier one */
                rl[r] = 0;
                int dup = 0; for (uint32_t k = 0; k < r; k++) if (rep[k] == rep[r]) dup = 1;
                if (!dup && p >= rep[r] + 1u) rl[r] = mlen(base, p - rep[r] - 1u, p, maxLen);
            }
            for (uint32_t t = 0; t < LZP_NCAND; t++) { cl[t] = LZP_CAND_LEN(c[t]); if (cl[t] > maxLen) cl[t] = maxLen; cd[t] = LZP_CAND_DIST(c[t]); }
            /* a long match ends the window: the path to here is committed and the match taken */
            uint32_t bl = 0, bd = 0, capped = 0;
            for (uint32_t r = 0; r < 4; r++) if (rl[r] > bl) { bl = rl[r]; bd = rep[r]; }
            for (uint32_t t = 0; t < LZP_NCAND; t++) if (cl[t] > bl) { bl = cl[t]; bd = cd[t]; capped = LZP_CAND_LEN(c[t]) == LZP_CAND_LENCAP; }
            if (bl >= LZP_NICE) { longLen = capped ? mlen(base, p - bd - 1u, p, maxLen) : bl; longDist = bd; break; }
            const uint32_t c0 = nd[i].cost, room = W - i;
            const uint32_t pm0 = lzm_price(PT, probs[LZM_ISMATCH + st * 16u + ps], 0), pm1 = lzm_price(PT, probs[LZM_ISMATCH + st * 16u + ps], 1);
            {   /* literal */
                const uint32_t cst = c0 + pm0 + lzm_price_literal(PT, probs, p, p ? base[p - 1] : 0u, base[p], st >= 7u, st >= 7u ? base[p - rep[0] - 1u] : 0u);
                if (cst < nd[i + 1].cost) { nd[i + 1].cost = cst; nd[i + 1].from = i; nd[i + 1].kind = K_LIT; nd[i + 1].len = 1; }
                if (end < i + 1) end = i + 1;
            }
            const uint32_t prep = pm1 + lzm_price(PT, probs[LZM_ISREP + st], 1);
            for (uint32_t r = 0; r < 4; r++) {
                const uint32_t L = rl[r] < room ? rl[r] : room;
                if (L < 2) continue;
                uint32_t sel;
                if (r == 0) sel = lzm_price(PT, probs[LZM_ISREPG0 + st], 0) + lzm_price(PT, probs[LZM_ISREP0LONG + st * 16u + ps], 1);
                else if (r == 1) sel = lzm_price(PT, probs[LZM_ISREPG0 + st], 1) + lzm_price(PT, probs[LZM_ISREPG1 + st], 0);
                else sel = lzm_price(PT, probs[LZM_ISREPG0 + st], 1) + lzm_price(PT, probs[LZM_ISREPG1 + st], 1) + lzm_price(PT, probs[LZM_ISREPG2 + st], r - 2u);
                for (uint32_t l = 2; l <= L; l++) {
                    const uint32_t cst = c0 + prep + sel + lzm_price_len(PT, probs + LZM_REPLEN, l, ps);
                    if (cst < nd[i + l].cost) { nd[i + l].cost = cst; nd[i + l].from = i; nd[i + l].kind = K_REP; nd[i + l].len = l; nd[i + l].dist = r; }
                }
                if (end < i + L) end = i + L;
            }
            {   /* matches: every length goes with the nearest candidate that reaches it */
                const uint32_t pmatch = pm1 + lzm_price(PT, probs[LZM_ISREP + st], 0);
                uint32_t ML = 0;
                for (uint32_t t = 0; t < LZP_NCAND; t++) if (cl[t] > ML) ML = cl[t];
                if (ML > room) ML = room;
                for (uint32_t l = 2; l <= ML; l++) {
                    uint32_t d = 0xFFFFFFFFu;
                    for (uint32_t t = 0; t < LZP_NCAND; t++) if (cl[t] >= l && cd[t] < d) d = cd[t];
                    int isrep = 0; for (uint32_t r = 0; r < 4; r++) if (rl[r] && rep[r] == d) isrep = 1;      /* stage R codes it as a rep: priced above */
                    if (isrep) continue;
                    const uint32_t cst = c0 + pmatch + lzm_price_len(PT, probs + LZM_LEN, l, ps) + lzm_price_dist(PT, probs, d, l - 2u < 4u ? l - 2u : 3u);
                    if (cst < nd[i + l].cost) { nd[i + l].cost = cst; nd[i + l].from = i; nd[i + l].kind = K_MATCH; nd[i + l].len = l; nd[i + l].dist = d; }
                }
                if (ML >= 2 && end < i + ML) end = i + ML;
            }
            i++;
        }
        /* commit the cheapest path to node i: its packets update the model as stage R will when it codes them */
        uint32_t np = 0;
        for (uint32_t j = i; j > 0; j = nd[j].from) path[np++] = j;
        while (np--) {
            const node_t *y = &nd[path[np]];
            const uint32_t p = pos + y->from;
            if (y->kind == K_LIT) commit_literal(probs, &x, base, p);
            else {
                const uint32_t d = y->kind == K_MATCH ? y->dist : x.rep[y->dist];
                lzm_commit_match(probs, &x, p, y->len, d);
                sink_match(sink, p, y->len, d);
            }
        }
        pos += i;
        if (longLen) { lzm_commit_match(probs, &x, pos, longLen, longDist); sink_match(sink, pos, longLen, longDist); pos += longLen; }
    }
    if (xOut) *xOut = x;
}

/* one frame -> per-block sequences (block-indexed arrays of the frame, layout of b2zo_zstd_find_sequences); cand = stage C's output */
void b2zo_lzma2_parse_frame(const void *basev, uint32_t n, const b2zo_enc_params *P, const uint32_t *cand, uint64_t *seqs, uint32_t *nseq) {
    const uint8_t *base = (const uint8_t *)basev;
    uint32_t *own = NULL;
    if (!cand) { own = (uint32_t *)malloc((size_t)n * LZP_NCAND * 4 + 4); b2zo_lzma2_candidates(base, n, P->frameLog, own); cand = own; }
    const uint32_t sliceBytes = B2Z_LZ2_SLICE_BLOCKS(P->frameLog, P->flags) * B2Z_BLOCK;
    uint16_t *probs = (uint16_t *)malloc(LZM_NPROBS * 2);
    const uint32_t nblk = (n + B2Z_BLOCK - 1) / B2Z_BLOCK;
    for (uint32_t b = 0; b < nblk; b++) nseq[b] = 0;
    for (uint32_t s0 = 0; s0 < n; s0 += sliceBytes) {             /* slices = stage R's state-reset chains: independent models */
        const uint32_t s1 = s0 + sliceBytes < n ? s0 + sliceBytes : n;
        sink_t sink = { seqs, nseq, s0 };
        parse_slice(base, s0, s1, cand, probs, &sink, NULL);
    }
    free(probs); free(own);
}

/* Test tap: the model stage P ends the frame's LAST slice with (see b2zo_lzma2_final_model) */
void b2zo_lzma2_parse_final_model(const void *basev, uint32_t n, const b2zo_enc_params *P, uint64_t *seqs, uint32_t *nseq, uint16_t *probsOut, uint32_t *ctxOut) {
    const uint8_t *base = (const uint8_t *)basev;
    uint32_t *cand = (uint32_t *)malloc((size_t)n * LZP_NCAND * 4 + 4);
    b2zo_lzma2_candidates(base, n, P->frameLog, cand);
    const uint32_t sliceBytes = B2Z_LZ2_SLICE_BLOCKS(P->frameLog, P->flags) * B2Z_BLOCK;
    const uint32_t nblk = (n + B2Z_BLOCK - 1) / B2Z_BLOCK;
    for (uint32_t b = 0; b < nblk; b++) nseq[b] = 0;
    lzm_ctx x; memset(&x, 0, sizeof(x));
    for (uint32_t s0 = 0; s0 < n; s0 += sliceBytes) {
        const uint32_t s1 = s0 + sliceBytes < n ? s0 + sliceBytes : n;
        sink_t sink = { seqs, nseq, s0 };
        parse_slice(base, s0, s1, cand, probsOut, &sink, &x);
    }
    ctxOut[0] = x.state; for (int i = 0; i < 4; i++) ctxOut[1 + i] = x.rep[i];
    free(cand);
}
