/* b2z_lzma_model.h -- the LZMA probability model as arithmetic: layout, bit prices, packet prices, packet updates.
 * Plain C, host + device (B2Z_HD).  Used by stage P (lzma2_parse.cu) and, read-only, by its sequential statement
 * (oracle/lzma2_opt_oracle.c) so that both price a packet the same way; stage R (lzma2_enc.cu) and the decoders keep their
 * own statements of the same model, and the reference decoder checks all of them.
 *
 * Format rules followed (reference, /root/reference/C/): probability sets and contexts LzmaEnc.c:2388-2600 / LzmaDec.c:130-227,
 * 11-bit adaptive probabilities with shift 5 (LzmaEnc.c:691-760), price = -log2(probability) in 1/16 bit, looked up from the
 * top 7 bits of the probability (the idea of LzmaEnc.c:2208-2232 ProbPrices; table values are ours, from the formula below). */
#ifndef B2Z_LZMA_MODEL_H
#define B2Z_LZMA_MODEL_H
#include "b2z_params.h"

/* model layout (uint16 probabilities), same offsets as b2z_lzma2.h / the oracle coders */
#define LZM_ISMATCH    0u      /* [12 states][16] */
#define LZM_ISREP      192u    /* [12] */
#define LZM_ISREPG0    204u
#define LZM_ISREPG1    216u
#define LZM_ISREPG2    228u
#define LZM_ISREP0LONG 240u    /* [12][16] */
#define LZM_POSSLOT    432u    /* [4 length states][64] */
#define LZM_SPECPOS    688u
#define LZM_ALIGN      804u
#define LZM_LEN        820u    /* choice, choice2, low[16][8], mid[16][8], high[256] */
#define LZM_REPLEN     1334u
#define LZM_LIT        1848u   /* [0x300 << (lc + lp)] */
#define LZM_L_CHOICE   0u
#define LZM_L_CHOICE2  1u
#define LZM_L_LOW      2u
#define LZM_L_MID      130u
#define LZM_L_HIGH     258u
/* the model at the compile-time context bits B2Z_LZ2_LC / LP / PB (the defaults, or what a statement compiled for one setting
 * defines them as) */
#define LZM_LITN       (0x300u << (B2Z_LZ2_LC + B2Z_LZ2_LP))
#define LZM_NPROBS     (LZM_LIT + LZM_LITN)
#define LZM_PBM        ((1u << B2Z_LZ2_PB) - 1u)
#define LZM_LPM        ((1u << B2Z_LZ2_LP) - 1u)

/* literal / position context bits of a coder (b2z_lz2_props: the LZMA2 properties byte).  Built from a constant byte, every
 * function below folds them into its code.  The *_p functions take them; the ones without the suffix use B2Z_LZ2_LC / LP / PB. */
typedef struct { uint32_t lc, lp, pb; } lzm_props;
B2Z_HD lzm_props lzm_props_of(uint32_t props) { lzm_props q; q.lc = b2z_lz2_lc(props); q.lp = b2z_lz2_lp(props); q.pb = b2z_lz2_pb(props); return q; }
B2Z_HD uint32_t lzm_litn(lzm_props q) { return 0x300u << (q.lc + q.lp); }
B2Z_HD uint32_t lzm_nprobs(lzm_props q) { return LZM_LIT + lzm_litn(q); }
B2Z_HD uint32_t lzm_pbm(lzm_props q) { return (1u << q.pb) - 1u; }
/* first probability of the literal coder of the byte at pos after byte prev */
B2Z_HD uint32_t lzm_lit_base(lzm_props q, uint32_t pos, uint32_t prev) { return LZM_LIT + 0x300u * (((pos & ((1u << q.lp) - 1u)) << q.lc) + (prev >> (8u - q.lc))); }

/* price[i] = round(-16 * log2((16 i + 8) / 2048)), i = probability >> 4 */
#define LZM_PRICE_LIST \
    128,103,91,83,77,73,69,65,63,60,58,56,54,52,50,49,47,46,45,43,42,41,40,39,38,37,36,35,35,34,33,32,32,31,30,30,29,28,28,27,27,26,25,25, \
    24,24,23,23,22,22,21,21,21,20,20,19,19,18,18,18,17,17,17,16,16,15,15,15,14,14,14,13,13,13,12,12,12,12,11,11,11,10,10,10,10,9,9,9,9,8,8,8, \
    7,7,7,7,7,6,6,6,6,5,5,5,5,4,4,4,4,4,3,3,3,3,3,2,2,2,2,2,1,1,1,1,1,0,0,0

/* stage P knobs (part of the algorithm: the oracle and the kernel must agree) */
#define LZP_WIN   256u     /* nodes of one dynamic-programme window (a window ends earlier where all paths meet)      */
#define LZP_NICE  32u      /* a match this long is taken at once: ends the window, never priced                      */
#define LZP_NCAND 4u       /* stage C candidates per position: nearest previous occurrence by 3-, 4-, 6-, 8-byte key */
#define LZP_CAND_LENCAP 255u   /* stage C stores min(length, 255); stage P extends a capped one when it takes it     */
#define LZP_PACK_CAND(dist, len) (((uint32_t)(dist) << 8) | (uint32_t)(len))   /* dist = distance - 1 (< 2^24), len 0 = none */
#define LZP_CAND_DIST(c) ((uint32_t)(c) >> 8)
#define LZP_CAND_LEN(c)  ((uint32_t)(c) & 0xFFu)

/* table t of stage C: key bytes and log2 of its entries for frames of 2^frameLog bytes */
B2Z_HD uint32_t lzp_key_bytes(uint32_t t) { return t == 0 ? 3u : (t == 1 ? 4u : (t == 2 ? 6u : 8u)); }
B2Z_HD uint32_t lzp_table_log(uint32_t t, uint32_t frameLog) {
    const uint32_t lo = 14u + 2u * t - (t == 3 ? 2u : (t == 2 ? 1u : 0u));      /* 14 16 17 18 */
    const uint32_t hi = lo + 4u;                                               /* 18 20 21 22 */
    const uint32_t want = frameLog - 4u + 2u * t - (t == 3 ? 2u : (t == 2 ? 1u : 0u));   /* frameLog-4, -2, -1, +0 */
    return want < lo ? lo : (want > hi ? hi : want);
}
B2Z_HD uint32_t lzp_table_index(uint64_t v /* 8 little-endian bytes at the position */, uint32_t keyBytes, uint32_t log) {
    return (uint32_t)(((v << (64u - 8u * keyBytes)) * B2Z_PRIME8) >> (64u - log));
}

B2Z_HD uint32_t lzm_price(const uint8_t *pt, uint32_t prob, uint32_t bit) { return pt[(prob ^ ((0u - bit) & 2047u)) >> 4]; }
B2Z_HD void lzm_update(uint16_t *p, uint32_t bit) { const uint32_t v = *p; *p = (uint16_t)(bit ? v - (v >> 5) : v + ((2048u - v) >> 5)); }

B2Z_HD uint32_t lzm_state_lit(uint32_t s) { return s < 4u ? 0u : (s < 10u ? s - 3u : s - 6u); }
B2Z_HD uint32_t lzm_state_match(uint32_t s) { return s < 7u ? 7u : 10u; }
B2Z_HD uint32_t lzm_state_rep(uint32_t s) { return s < 7u ? 8u : 11u; }

B2Z_HD uint32_t lzm_dist_slot(uint32_t dist) {
    if (dist < 4u) return dist;
#ifdef __CUDA_ARCH__
    const uint32_t nb = 31u - (uint32_t)__clz((int)dist);
#else
    const uint32_t nb = 31u - (uint32_t)__builtin_clz(dist);
#endif
    return (nb << 1) | ((dist >> (nb - 1u)) & 1u);
}

/* ---- prices: pure functions of the model */
B2Z_HD uint32_t lzm_price_tree(const uint8_t *pt, const uint16_t *p, uint32_t bits, uint32_t v) {
    uint32_t m = 1, c = 0;
    for (uint32_t i = bits; i--;) { const uint32_t b = (v >> i) & 1u; c += lzm_price(pt, p[m], b); m = (m << 1) | b; }
    return c;
}
B2Z_HD uint32_t lzm_price_tree_rev(const uint8_t *pt, const uint16_t *p, uint32_t bits, uint32_t v) {
    uint32_t m = 1, c = 0;
    for (uint32_t i = 0; i < bits; i++) { const uint32_t b = (v >> i) & 1u; c += lzm_price(pt, p[m], b); m = (m << 1) | b; }
    return c;
}
B2Z_HD uint32_t lzm_price_len(const uint8_t *pt, const uint16_t *l, uint32_t len, uint32_t ps) {
    len -= 2u;
    if (len < 8u) return lzm_price(pt, l[LZM_L_CHOICE], 0) + lzm_price_tree(pt, l + LZM_L_LOW + ps * 8u, 3, len);
    if (len < 16u) return lzm_price(pt, l[LZM_L_CHOICE], 1) + lzm_price(pt, l[LZM_L_CHOICE2], 0) + lzm_price_tree(pt, l + LZM_L_MID + ps * 8u, 3, len - 8u);
    return lzm_price(pt, l[LZM_L_CHOICE], 1) + lzm_price(pt, l[LZM_L_CHOICE2], 1) + lzm_price_tree(pt, l + LZM_L_HIGH, 8, len - 16u);
}
/* distance (= distance - 1) coded after a length of length-state ls = min(len - 2, 3) */
B2Z_HD uint32_t lzm_price_dist(const uint8_t *pt, const uint16_t *probs, uint32_t dist, uint32_t ls) {
    const uint32_t slot = lzm_dist_slot(dist);
    uint32_t c = lzm_price_tree(pt, probs + LZM_POSSLOT + ls * 64u, 6, slot);
    if (slot >= 4u) {
        const uint32_t fb = (slot >> 1) - 1u, b = (2u | (slot & 1u)) << fb, red = dist - b;
        if (slot < 14u) c += lzm_price_tree_rev(pt, probs + LZM_SPECPOS + b - slot - 1u, fb, red);
        else c += (fb - 4u) * 16u + lzm_price_tree_rev(pt, probs + LZM_ALIGN, 4, red & 15u);
    }
    return c;
}
/* the 8 bits of literal `sym` at pos after byte `prev`; matched = coded in a state >= 7 against byte mb (the byte at rep0) */
B2Z_HD uint32_t lzm_price_literal_p(const uint8_t *pt, const uint16_t *probs, lzm_props q, uint32_t pos, uint32_t prev, uint32_t sym, uint32_t matched, uint32_t mb) {
    const uint16_t *p = probs + lzm_lit_base(q, pos, prev);
    uint32_t c = 0, m = 1;
    for (uint32_t i = 8; i--;) {
        const uint32_t b = (sym >> i) & 1u;
        if (matched) { const uint32_t mbit = (mb >> i) & 1u; c += lzm_price(pt, p[((1u + mbit) << 8) + m], b); if (mbit != b) matched = 0; }
        else c += lzm_price(pt, p[m], b);
        m = (m << 1) | b;
    }
    return c;
}
B2Z_HD uint32_t lzm_price_literal(const uint8_t *pt, const uint16_t *probs, uint32_t pos, uint32_t prev, uint32_t sym, uint32_t matched, uint32_t mb) {
    return lzm_price_literal_p(pt, probs, lzm_props_of(B2Z_LZ2_PROPS), pos, prev, sym, matched, mb);
}

/* ---- the probability updates of one coded packet (what stage R does to its model while it codes the packet) */
B2Z_HD void lzm_update_tree(uint16_t *p, uint32_t bits, uint32_t v) { uint32_t m = 1; for (uint32_t i = bits; i--;) { const uint32_t b = (v >> i) & 1u; lzm_update(p + m, b); m = (m << 1) | b; } }
B2Z_HD void lzm_update_tree_rev(uint16_t *p, uint32_t bits, uint32_t v) { uint32_t m = 1; for (uint32_t i = 0; i < bits; i++) { const uint32_t b = (v >> i) & 1u; lzm_update(p + m, b); m = (m << 1) | b; } }
B2Z_HD void lzm_update_len(uint16_t *l, uint32_t len, uint32_t ps) {
    len -= 2u;
    if (len < 8u) { lzm_update(l + LZM_L_CHOICE, 0); lzm_update_tree(l + LZM_L_LOW + ps * 8u, 3, len); }
    else if (len < 16u) { lzm_update(l + LZM_L_CHOICE, 1); lzm_update(l + LZM_L_CHOICE2, 0); lzm_update_tree(l + LZM_L_MID + ps * 8u, 3, len - 8u); }
    else { lzm_update(l + LZM_L_CHOICE, 1); lzm_update(l + LZM_L_CHOICE2, 1); lzm_update_tree(l + LZM_L_HIGH, 8, len - 16u); }
}
typedef struct { uint32_t state, rep[4]; } lzm_ctx;      /* coder state next to the probabilities */

B2Z_HD void lzm_commit_literal_p(uint16_t *probs, lzm_ctx *x, lzm_props q, uint32_t pos, uint32_t prev, uint32_t sym, uint32_t mb /* byte at rep0, used when state >= 7 */) {
    lzm_update(probs + LZM_ISMATCH + x->state * 16u + (pos & lzm_pbm(q)), 0);
    uint16_t *p = probs + lzm_lit_base(q, pos, prev);
    uint32_t m = 1, matched = x->state >= 7u;
    for (uint32_t i = 8; i--;) {
        const uint32_t b = (sym >> i) & 1u;
        if (matched) { const uint32_t mbit = (mb >> i) & 1u; lzm_update(p + ((1u + mbit) << 8) + m, b); if (mbit != b) matched = 0; }
        else lzm_update(p + m, b);
        m = (m << 1) | b;
    }
    x->state = lzm_state_lit(x->state);
}
/* a match of len (2..273) at dist (= distance - 1): coded as the first rep that holds dist, else as a new distance (stage R's rule) */
B2Z_HD void lzm_commit_match_p(uint16_t *probs, lzm_ctx *x, lzm_props q, uint32_t pos, uint32_t len, uint32_t dist) {
    const uint32_t ps = pos & lzm_pbm(q), s = x->state;
    lzm_update(probs + LZM_ISMATCH + s * 16u + ps, 1);
    const int r = dist == x->rep[0] ? 0 : (dist == x->rep[1] ? 1 : (dist == x->rep[2] ? 2 : (dist == x->rep[3] ? 3 : -1)));
    if (r < 0) {
        lzm_update(probs + LZM_ISREP + s, 0);
        lzm_update_len(probs + LZM_LEN, len, ps);
        const uint32_t slot = lzm_dist_slot(dist);
        lzm_update_tree(probs + LZM_POSSLOT + (len - 2u < 4u ? len - 2u : 3u) * 64u, 6, slot);
        if (slot >= 4u) {
            const uint32_t fb = (slot >> 1) - 1u, b = (2u | (slot & 1u)) << fb, red = dist - b;
            if (slot < 14u) lzm_update_tree_rev(probs + LZM_SPECPOS + b - slot - 1u, fb, red);
            else lzm_update_tree_rev(probs + LZM_ALIGN, 4, red & 15u);
        }
        x->rep[3] = x->rep[2]; x->rep[2] = x->rep[1]; x->rep[1] = x->rep[0]; x->rep[0] = dist;
        x->state = lzm_state_match(s);
    } else {
        lzm_update(probs + LZM_ISREP + s, 1);
        if (r == 0) { lzm_update(probs + LZM_ISREPG0 + s, 0); lzm_update(probs + LZM_ISREP0LONG + s * 16u + ps, 1); }
        else {
            lzm_update(probs + LZM_ISREPG0 + s, 1);
            if (r == 1) lzm_update(probs + LZM_ISREPG1 + s, 0);
            else { lzm_update(probs + LZM_ISREPG1 + s, 1); lzm_update(probs + LZM_ISREPG2 + s, (uint32_t)(r - 2)); }
            if (r == 3) x->rep[3] = x->rep[2];
            if (r >= 2) x->rep[2] = x->rep[1];
            x->rep[1] = x->rep[0]; x->rep[0] = dist;
        }
        lzm_update_len(probs + LZM_REPLEN, len, ps);
        x->state = lzm_state_rep(s);
    }
}

B2Z_HD void lzm_commit_literal(uint16_t *probs, lzm_ctx *x, uint32_t pos, uint32_t prev, uint32_t sym, uint32_t mb) {
    lzm_commit_literal_p(probs, x, lzm_props_of(B2Z_LZ2_PROPS), pos, prev, sym, mb);
}
B2Z_HD void lzm_commit_match(uint16_t *probs, lzm_ctx *x, uint32_t pos, uint32_t len, uint32_t dist) { lzm_commit_match_p(probs, x, lzm_props_of(B2Z_LZ2_PROPS), pos, len, dist); }

#endif
