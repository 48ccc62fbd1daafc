/* zstd_opt_oracle.c -- sequential statement of the price-based parse of the GPU Zstandard encoder (stage Z; flag B2Z_FLAG_ZSTD_OPT).
 *
 * TEST INFRASTRUCTURE ONLY (see oracle.h).  States what csrc/zstd_enc_parse.cu computes for one frame: per 128 KiB block, the
 * sequences and literal bytes stage E codes (same arrays as stage M, b2zo_zstd_find_sequences).
 *
 *   candidates  stage C's words (lzma2_opt_oracle.c: nearest previous occurrence by 3/4/6/8-byte keys), shared with method 21.
 *   parse       one chain per BLOCK: a forward dynamic programme over windows of <= LZP_WIN positions; node i = cheapest known
 *               coding of the window's first i bytes + the state it leaves (repcode history, literals since the last match);
 *               edges: literal (priced from the block's byte histogram), repcode matches, candidate matches (every length goes
 *               with the nearest candidate that reaches it), priced from adaptive counts of the offset / match-length /
 *               literal-length codes the block has produced so far (b2z_zstd_cost.h).  A window ends where all paths meet, at
 *               LZP_WIN nodes, or at a match of >= LZP_NICE bytes, which is taken at once.
 *   Role in the reference: zstd_opt.c:1077 ZSTD_compressBlock_opt_generic (levels 16-22) with :590 ZSTD_insertBtAndGetAllMatches
 *   and the price functions :295-356 -- same idea; this formulation, its statistics and its numbers are ours.
 */
#include <stdlib.h>
#include <string.h>
#include "oracle.h"
#include "b2z_params.h"
#include "b2z_lzma_model.h"      /* LZP_* : stage C word layout, window size, nice length */
#include "b2z_zstd_cost.h"

static const zop_tables ZT = ZOP_TABLES_INIT;

static uint32_t mlen(const uint8_t *b, uint32_t q, uint32_t p, uint32_t maxLen) { uint32_t l = 0; while (l < maxLen && b[q + l] == b[p + l]) l++; return l; }

enum { K_LIT = 0, K_MATCH = 1 };
typedef struct { uint32_t cost, from, kind, len, off; zop_ctx x; } znode;

static void parse_block(const uint8_t *base, uint32_t b0, uint32_t b1, const uint32_t *cand, uint64_t *seqs, uint32_t *nseqOut, uint8_t *lits, uint32_t *nlitOut) {
    znode nd[LZP_WIN + 1];
    uint32_t path[LZP_WIN + 1];
    uint32_t litPrice[256], hist[256];
    zop_stats st;
    memset(hist, 0, sizeof(hist));
    for (uint32_t p = b0; p < b1; p++) hist[base[p]]++;
    for (uint32_t k = 0; k < 256; k++) litPrice[k] = hist[k] ? zop_cost(&ZT, hist[k], b1 - b0) : 0;      /* static per block (adaptive literal counts gain nothing on G2: tried) */
    for (uint32_t k = 0; k < ZOP_N_OF; k++) st.of[k] = 1;
    for (uint32_t k = 0; k < ZOP_N_ML; k++) st.ml[k] = 1;
    for (uint32_t k = 0; k < ZOP_N_LL; k++) st.ll[k] = 1;
    st.ofSum = ZOP_N_OF; st.mlSum = ZOP_N_ML; st.llSum = ZOP_N_LL;
    zop_ctx x; x.rep[0] = x.rep[1] = x.rep[2] = 0; x.litLen = 0;
    uint32_t nseq = 0, nlit = 0, pos = b0;
    while (pos < b1) {
        const uint32_t W = (b1 - pos) < LZP_WIN ? (b1 - pos) : LZP_WIN;
        nd[0].cost = 0; nd[0].x = x;
        for (uint32_t j = 1; j <= W; j++) nd[j].cost = 0xFFFFFFFFu;
        uint32_t end = 0, i = 0, longLen = 0, longOff = 0;
        for (;;) {
            if (i) {
                znode *y = &nd[i]; const znode *f = &nd[y->from];
                y->x = f->x;
                if (y->kind == K_LIT) y->x.litLen = f->x.litLen + 1; else zop_after_match(&y->x, y->off);
            }
            if (i == W || (i && i == end)) break;
            const uint32_t p = pos + i, maxLen = b1 - p, room = W - i;
            const zop_ctx *cx = &nd[i].x;
            const uint32_t *c = cand + (size_t)p * LZP_NCAND;
            /* repcode offsets as the next sequence would see them (shifted when no literal precedes it) */
            uint32_t ro[3], rl[3];
            if (cx->litLen) { ro[0] = cx->rep[0]; ro[1] = cx->rep[1]; ro[2] = cx->rep[2]; }
            else { ro[0] = cx->rep[1]; ro[1] = cx->rep[2]; ro[2] = cx->rep[0] > 1 ? cx->rep[0] - 1 : 0; }
            for (uint32_t r = 0; r < 3; r++) {
                rl[r] = 0;
                int dup = 0; for (uint32_t k = 0; k < r; k++) if (ro[k] == ro[r]) dup = 1;
                if (ro[r] && !dup && p >= ro[r]) rl[r] = mlen(base, p - ro[r], p, maxLen);
            }
            uint32_t cl[LZP_NCAND], co[LZP_NCAND];
            for (uint32_t t = 0; t < LZP_NCAND; t++) { cl[t] = LZP_CAND_LEN(c[t]); if (cl[t] > maxLen) cl[t] = maxLen; co[t] = LZP_CAND_DIST(c[t]) + 1; }
            uint32_t bl = 0, bo = 0, capped = 0;
            for (uint32_t r = 0; r < 3; r++) if (rl[r] > bl) { bl = rl[r]; bo = ro[r]; }
            for (uint32_t t = 0; t < LZP_NCAND; t++) if (cl[t] > bl) { bl = cl[t]; bo = co[t]; capped = LZP_CAND_LEN(c[t]) == LZP_CAND_LENCAP; }
            if (bl >= LZP_NICE) { longLen = capped ? mlen(base, p - bo, p, maxLen) : bl; longOff = bo; break; }
            const uint32_t c0 = nd[i].cost;
            {   /* literal */
                const uint32_t cst = c0 + litPrice[base[p]];
                if (cst < nd[i + 1].cost) { nd[i + 1].cost = cst; nd[i + 1].from = i; nd[i + 1].kind = K_LIT; nd[i + 1].len = 1; }
                if (end < i + 1) end = i + 1;
            }
            for (uint32_t r = 0; r < 3; r++) {
                const uint32_t L = rl[r] < room ? rl[r] : room;
                if (L < ZOP_MINMATCH) continue;
                const uint32_t ob = zop_off_base(cx, ro[r]);
                for (uint32_t l = ZOP_MINMATCH; l <= L; l++) {
                    const uint32_t cst = c0 + zop_seq_price(&ZT, &st, cx->litLen, ob, l);
                    if (cst < nd[i + l].cost) { nd[i + l].cost = cst; nd[i + l].from = i; nd[i + l].kind = K_MATCH; nd[i + l].len = l; nd[i + l].off = ro[r]; }
                }
                if (end < i + L) end = i + L;
            }
            {
                uint32_t ML = 0;
                for (uint32_t t = 0; t < LZP_NCAND; t++) if (cl[t] > ML) ML = cl[t];
                if (ML > room) ML = room;
                for (uint32_t l = ZOP_MINMATCH; l <= ML; l++) {
                    uint32_t o = 0xFFFFFFFFu;
                    for (uint32_t t = 0; t < LZP_NCAND; t++) if (cl[t] >= l && co[t] < o) o = co[t];
                    const uint32_t cst = c0 + zop_seq_price(&ZT, &st, cx->litLen, zop_off_base(cx, o), l);
                    if (cst < nd[i + l].cost) { nd[i + l].cost = cst; nd[i + l].from = i; nd[i + l].kind = K_MATCH; nd[i + l].len = l; nd[i + l].off = o; }
                }
                if (ML >= ZOP_MINMATCH && end < i + ML) end = i + ML;
            }
            i++;
        }
        uint32_t np = 0;
        for (uint32_t j = i; j > 0; j = nd[j].from) path[np++] = j;
        for (;;) {
            uint32_t p, len, off;
            if (np) { const znode *y = &nd[path[--np]]; p = pos + y->from; if (y->kind == K_LIT) { lits[nlit++] = base[p]; x.litLen++; continue; } len = y->len; off = y->off; }
            else if (longLen) { p = pos + i; len = longLen; off = longOff; longLen = 0; i += len; }
            else break;
            if (nseq >= B2Z_MAXSEQ) { for (uint32_t k = 0; k < len; k++) lits[nlit++] = base[p + k]; x.litLen += len; continue; }   /* array full: the bytes stay literals */
            const uint32_t ob = zop_off_base(&x, off);
            zop_count_seq(&ZT, &st, x.litLen, ob, len);
            seqs[nseq++] = B2Z_PACK_SEQ(ob, x.litLen, len);
            zop_after_match(&x, off);
        }
        pos += i;
    }
    *nseqOut = nseq; *nlitOut = nlit;
}

/* one frame -> per-block sequences + literal bytes (arrays of the frame, block-indexed; lits at the block's offset) */
void b2zo_zstd_parse_frame(const void *basev, uint32_t n, const b2zo_enc_params *P, const uint32_t *cand, uint64_t *seqs, uint32_t *nseq, uint8_t *lits, uint32_t *nlit) {
    const uint8_t *base = (const uint8_t *)basev;
    uint32_t *own = NULL;
    if (!cand) { own = (uint32_t *)malloc((size_t)n * LZP_NCAND * 4 + 4); b2zo_lzma2_candidates(base, n, P->frameLog, own); cand = own; }
    const uint32_t nblk = (n + B2Z_BLOCK - 1) / B2Z_BLOCK;
    for (uint32_t b = 0; b < nblk; b++) {
        const uint32_t b0 = b * B2Z_BLOCK, b1 = b0 + B2Z_BLOCK < n ? b0 + B2Z_BLOCK : n;
        parse_block(base, b0, b1, cand, seqs + (size_t)b * B2Z_MAXSEQ, nseq + b, lits + b0, nlit + b);
    }
    free(own);
}
