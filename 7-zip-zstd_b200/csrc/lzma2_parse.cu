// lzma2_parse.cu -- the price-based parse of the block-parallel LZMA2 encoder (7-Zip method 21, flag B2Z_FLAG_LZ2_OPT) for sm_90a.
//
// Two kernels in front of stage R (lzma2_enc.cu), replacing the greedy stage M for this mode:
//
//   stage C  lzma2_cand_kernel -- one warp per frame, 32 positions per step.  For every position and each of four direct-mapped
//            tables (keys of 3, 4, 6 and 8 bytes) the NEAREST earlier position whose key falls into the same table entry, and the
//            common-prefix length with it: LZP_NCAND packed words per position.  Lanes of one step that hit the same entry are
//            resolved with __match_any_sync (a lane takes the highest lower lane of its group, the group's highest lane writes
//            the entry), so the result is the pure function the oracle states position by position.
//            Role in the reference: the finders that give the optimal parsers their (length, nearest distance) pairs --
//            LzFind.c:1219 (Bt4_MatchFinder_GetMatches), fast-lzma2/radix_get.h:84 (RMF_getMatch).
//   stage P  lzma2_parse_kernel -- one warp per state-reset slice (the chains of stage R).  A forward dynamic programme over
//            windows of <= LZP_WIN positions held in shared memory: node i = cheapest known coding of the window's first i bytes
//            + the coder state it leaves.  Lanes price the edges of a node in parallel (lane = match length; the 8 bits of a
//            literal), prices come from the slice's adaptive model in shared memory as it stands at the window start; the chosen
//            packets then update that model exactly as stage R will when it codes them (lzm_commit_*, b2z_lzma_model.h).
//            Role in the reference: LzmaEnc.c:1225 (GetOptimum), fast-lzma2/lzma2_enc.c:949 (LZMA_optimalParse).
//   Output: per-block sequences (literal run, match length, distance) in the arrays stage R already reads.
//
// Oracle statement: oracle/lzma2_opt_oracle.c (candidates and sequences must be identical).
#include "b2z_device.cuh"
#include "b2z_kernels.h"
#include "b2z_lzma2.h"
#include "b2z_lzma_model.h"

namespace b2z {

// ------------------------------------------------------------------------------------------------------------ stage C
__host__ __device__ inline uint32_t lzma2_cand_table_words(uint32_t frameLog) {
    uint32_t w = 0;
    for (uint32_t t = 0; t < LZP_NCAND; t++) w += 1u << lzp_table_log(t, frameLog);
    return w;
}

__global__ void __launch_bounds__(32)
lzma2_cand_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, uint32_t* __restrict__ tables, uint32_t* __restrict__ cand) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warpSlot = blockIdx.x, nWarps = gridDim.x;
    const uint64_t F = 1ull << g.frameLog;
    const uint64_t nFrames = (srcSize + F - 1) >> g.frameLog;
    const uint32_t tableWords = lzma2_cand_table_words(g.frameLog);
    uint32_t* const T0 = tables + (size_t)warpSlot * tableWords;
    uint32_t lg[LZP_NCAND], toff[LZP_NCAND];
    {
        uint32_t o = 0;
#pragma unroll
        for (uint32_t t = 0; t < LZP_NCAND; t++) { lg[t] = lzp_table_log(t, g.frameLog); toff[t] = o; o += 1u << lg[t]; }
    }
    const uint32_t ltMask = (1u << lane) - 1u;

    for (uint64_t f = warpSlot; f < nFrames; f += nWarps) {
        const uint64_t f0 = f << g.frameLog;
        const uint32_t n = enc_frame_bytes(g, srcSize, f);
        const uint64_t* __restrict__ w = reinterpret_cast<const uint64_t*>(src + f0);
        const uint32_t nWords = (n + 7u) >> 3;
        {
            uint4* t4 = reinterpret_cast<uint4*>(T0);
            const uint4 z = make_uint4(0, 0, 0, 0);
            for (uint32_t i = lane; i < tableWords / 4u; i += 32u) __stcg(t4 + i, z);
            __syncwarp();
        }
        uint4* const out = reinterpret_cast<uint4*>(cand) + f0;
        for (uint32_t base = 0; base < n; base += 32u) {
            const uint32_t p = base + lane;
            const bool live = p < n;
            const uint64_t v = live ? ld64u(w, p, nWords) : 0ull;
            uint32_t q1[LZP_NCAND], idx[LZP_NCAND]; bool writer[LZP_NCAND];
            // ---- read phase: the entry as the previous steps left it, or the nearest lower lane of this step with the same entry
#pragma unroll
            for (uint32_t t = 0; t < LZP_NCAND; t++) {
                const bool valid = live && p + lzp_key_bytes(t) <= n;
                idx[t] = lzp_table_index(v, lzp_key_bytes(t), lg[t]);
                const uint32_t grp = __match_any_sync(B2Z_FULL, valid ? idx[t] : (0x80000000u | lane));
                const uint32_t lower = grp & ltMask;
                q1[t] = 0; writer[t] = false;
                if (valid) {
                    q1[t] = lower ? base + (31u - (uint32_t)__clz((int)lower)) + 1u : __ldcg(T0 + toff[t] + idx[t]);
                    writer[t] = (grp >> lane) == 1u;                 // no higher lane in the group
                }
            }
            __syncwarp();
            // ---- write phase: the newest position of every entry touched by this step
#pragma unroll
            for (uint32_t t = 0; t < LZP_NCAND; t++) if (writer[t]) __stcg(T0 + toff[t] + idx[t], p + 1u);
            // ---- verify: common-prefix length with each candidate
            uint32_t c[LZP_NCAND];
            const uint32_t maxLen = live ? ((n - p) < B2Z_LZ2_MAXLEN ? (n - p) : B2Z_LZ2_MAXLEN) : 0u;
#pragma unroll
            for (uint32_t t = 0; t < LZP_NCAND; t++) {
                c[t] = 0;
                if (q1[t]) {
                    const uint32_t l = match_len_pv(w, q1[t] - 1u, p, v, maxLen, nWords);
                    if (l >= 2u) c[t] = LZP_PACK_CAND(p - q1[t], l < LZP_CAND_LENCAP ? l : LZP_CAND_LENCAP);
                }
            }
            if (live) __stcs(out + p, make_uint4(c[0], c[1], c[2], c[3]));
            __syncwarp();                                            // this step's entries are visible to the next step's reads
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------------------ stage P
enum : uint32_t { PK_LIT = 0, PK_REP = 1, PK_MATCH = 2 };
#define PLINK(from, len, kind, r) ((from) | ((len) << 9) | ((kind) << 18) | ((r) << 20))
#define PLINK_FROM(x) ((x) & 0x1FFu)
#define PLINK_LEN(x)  (((x) >> 9) & 0x1FFu)
#define PLINK_KIND(x) (((x) >> 18) & 3u)
#define PLINK_R(x)    (((x) >> 20) & 3u)

__constant__ uint8_t c_lzm_prices[128] = { LZM_PRICE_LIST };

struct ParseSmem {                       // one warp's working set; the model, lzm_nprobs() probabilities, follows it
    uint32_t cost[LZP_WIN + 1];
    uint32_t link[LZP_WIN + 1];          // best arrival: PLINK(from, len, kind, rep index)
    uint32_t dist[LZP_WIN + 1];          // ... its distance - 1 (PK_MATCH)
    uint32_t rep[LZP_WIN + 1][4];        // coder state the best arrival leaves
    uint4    cand[LZP_WIN];              // stage C's words of the window's positions
    uint16_t path[LZP_WIN + 1];
    uint8_t  state[LZP_WIN + 1];
    uint8_t  litMb[LZP_WIN + 1];         // byte at rep0 of the node (the matched-literal context), kept for the commit
    uint8_t  win[LZP_WIN + 40];          // win[k] = frame byte pos - 1 + k
    uint8_t  pt[128];
    uint32_t ctx[5];                     // committed coder state: state, rep0..3
};
size_t lzma2_parse_smem_bytes(uint32_t flags) { return sizeof(ParseSmem) + (size_t)lzm_nprobs(lzm_props_of(b2z_lz2_props(flags))) * sizeof(uint16_t); }

// DYN: lc / lp / pb from the properties byte in g.flags (B2Z_FLAG_LZ2_PROPS); otherwise the defaults, as compile-time constants
template <bool DYN = false>
__global__ void __launch_bounds__(32)
lzma2_parse_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, const uint32_t* __restrict__ cand,
                   uint64_t* __restrict__ seqs, uint32_t* __restrict__ nseq, uint32_t nChains) {
    B2Z_DYN_SMEM(ParseSmem, S);
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t chain = blockIdx.x;
    if (chain >= nChains) return;
    const uint64_t F = 1ull << g.frameLog;
    const uint32_t bpf = (uint32_t)(F >> 17), sliceBlocks = B2Z_LZ2_SLICE_BLOCKS(g.frameLog, g.flags), spf = bpf / sliceBlocks;
    const uint32_t f = chain / spf, sl = chain - f * spf;
    const uint64_t f0 = (uint64_t)f << g.frameLog;
    const uint32_t n = (uint32_t)((srcSize - f0) < F ? (srcSize - f0) : F);
    const uint32_t s0 = sl * sliceBlocks * B2Z_BLOCK;
    if (s0 >= n) return;                                            // slice beyond the end of a short last frame (its nseq stay 0)
    const uint32_t s1 = (s0 + sliceBlocks * B2Z_BLOCK) < n ? (s0 + sliceBlocks * B2Z_BLOCK) : n;
    const uint8_t* __restrict__ base = src + f0;
    const uint4* __restrict__ cand4 = reinterpret_cast<const uint4*>(cand) + f0;
    uint64_t* const fseqs = seqs + (size_t)f * bpf * B2Z_MAXSEQ;
    uint32_t* const fnseq = nseq + (size_t)f * bpf;
    const uint8_t* const pt = S->pt;
    uint16_t* const probs = reinterpret_cast<uint16_t*>(S + 1);
    const lzm_props q = lzm_props_of(DYN ? b2z_lz2_props(g.flags) : B2Z_LZ2_PROPS);

    for (uint32_t k = lane; k < 128u; k += 32u) S->pt[k] = c_lzm_prices[k];
    for (uint32_t k = lane; k < lzm_nprobs(q); k += 32u) probs[k] = 1024;
    if (lane < 5u) S->ctx[lane] = 0;
    __syncwarp();

    // lane 0's sink: sequences of the block being filled
    uint32_t prevEnd = s0, curBlk = s0 >> 17, cnt = 0;
    auto sink = [&](uint32_t pos, uint32_t len, uint32_t dist) {     // lane 0 only
        const uint32_t b = pos >> 17;
        if (b != curBlk) { fnseq[curBlk] = cnt; curBlk = b; cnt = 0; }
        if (cnt >= B2Z_MAXSEQ) return;
        const uint32_t bs = b << 17, from = prevEnd > bs ? prevEnd : bs;
        fseqs[(size_t)b * B2Z_MAXSEQ + cnt++] = B2Z_PACK_SEQ(dist + 1u + 3u, pos - from, len);
        prevEnd = pos + len;
    };

    uint32_t pos = s0;
    while (pos < s1) {
        const uint32_t W = (s1 - pos) < LZP_WIN ? (s1 - pos) : LZP_WIN;
        // ---- stage the window: bytes pos-1 .. pos+W+32 (zero past the slice end / before the frame), candidates, node costs
        for (uint32_t k = lane; k < W + 34u; k += 32u) {
            const uint32_t a = pos + k;                              // frame byte a - 1
            S->win[k] = (a >= 1u && a - 1u < s1) ? __ldg(base + a - 1u) : (uint8_t)0;
        }
        for (uint32_t k = lane; k < W; k += 32u) S->cand[k] = __ldg(cand4 + pos + k);
        for (uint32_t k = lane; k <= W; k += 32u) S->cost[k] = k ? 0xFFFFFFFFu : 0u;
        if (lane == 0) { S->state[0] = (uint8_t)S->ctx[0]; S->rep[0][0] = S->ctx[1]; S->rep[0][1] = S->ctx[2]; S->rep[0][2] = S->ctx[3]; S->rep[0][3] = S->ctx[4]; }
        __syncwarp();

        uint32_t end = 0, i = 0, longLen = 0, longDist = 0;
        uint32_t st = S->ctx[0], r0 = S->ctx[1], r1 = S->ctx[2], r2 = S->ctx[3], r3 = S->ctx[4];     // state of node i (warp-uniform)
        for (;;) {
            if (i) {                                                 // node i is final: the coder state its best arrival leaves
                const uint32_t lk = S->link[i], fr = PLINK_FROM(lk), kind = PLINK_KIND(lk);
                const uint32_t fs = S->state[fr], a0 = S->rep[fr][0], a1 = S->rep[fr][1], a2 = S->rep[fr][2], a3 = S->rep[fr][3];
                if (kind == PK_LIT) { st = lzm_state_lit(fs); r0 = a0; r1 = a1; r2 = a2; r3 = a3; }
                else if (kind == PK_REP) {
                    const uint32_t r = PLINK_R(lk);
                    st = lzm_state_rep(fs);
                    if (r == 0u) { r0 = a0; r1 = a1; r2 = a2; r3 = a3; }
                    else if (r == 1u) { r0 = a1; r1 = a0; r2 = a2; r3 = a3; }
                    else if (r == 2u) { r0 = a2; r1 = a0; r2 = a1; r3 = a3; }
                    else { r0 = a3; r1 = a0; r2 = a1; r3 = a2; }
                } else { st = lzm_state_match(fs); r0 = S->dist[i]; r1 = a0; r2 = a1; r3 = a2; }
                if (lane == 0) { S->state[i] = (uint8_t)st; S->rep[i][0] = r0; S->rep[i][1] = r1; S->rep[i][2] = r2; S->rep[i][3] = r3; }
            }
            if (i == W || (i && i == end)) break;
            const uint32_t p = pos + i, ps = p & lzm_pbm(q);
            const uint32_t maxLen = (s1 - p) < B2Z_LZ2_MAXLEN ? (s1 - p) : B2Z_LZ2_MAXLEN;
            const uint32_t lim32 = maxLen < 32u ? maxLen : 32u;
            const uint32_t curB = S->win[i + 1u + lane];             // frame byte p + lane (zero past the slice end: never compared there)
            // ---- rep lengths: lane k compares byte k; a rep equal to an earlier one is the earlier one
            uint32_t rl0 = 0, rl1 = 0, rl2 = 0, rl3 = 0;
            {
                const bool v0 = p >= r0 + 1u, v1 = r1 != r0 && p >= r1 + 1u, v2 = r2 != r0 && r2 != r1 && p >= r2 + 1u,
                           v3 = r3 != r0 && r3 != r1 && r3 != r2 && p >= r3 + 1u;
                const uint32_t b0 = (v0 && lane < lim32) ? (uint32_t)__ldg(base + p - r0 - 1u + lane) : 256u;
                const uint32_t b1 = (v1 && lane < lim32) ? (uint32_t)__ldg(base + p - r1 - 1u + lane) : 256u;
                const uint32_t b2 = (v2 && lane < lim32) ? (uint32_t)__ldg(base + p - r2 - 1u + lane) : 256u;
                const uint32_t b3 = (v3 && lane < lim32) ? (uint32_t)__ldg(base + p - r3 - 1u + lane) : 256u;
                const uint32_t m0 = __ballot_sync(B2Z_FULL, b0 != curB), m1 = __ballot_sync(B2Z_FULL, b1 != curB),
                               m2 = __ballot_sync(B2Z_FULL, b2 != curB), m3 = __ballot_sync(B2Z_FULL, b3 != curB);
                rl0 = m0 ? (uint32_t)(__ffs((int)m0) - 1) : 32u; rl1 = m1 ? (uint32_t)(__ffs((int)m1) - 1) : 32u;
                rl2 = m2 ? (uint32_t)(__ffs((int)m2) - 1) : 32u; rl3 = m3 ? (uint32_t)(__ffs((int)m3) - 1) : 32u;
                if (rl0 == 32u && maxLen > 32u) rl0 = warp_extend(base, p - r0 - 1u, p, 32u, maxLen, lane);
                if (rl1 == 32u && maxLen > 32u) rl1 = warp_extend(base, p - r1 - 1u, p, 32u, maxLen, lane);
                if (rl2 == 32u && maxLen > 32u) rl2 = warp_extend(base, p - r2 - 1u, p, 32u, maxLen, lane);
                if (rl3 == 32u && maxLen > 32u) rl3 = warp_extend(base, p - r3 - 1u, p, 32u, maxLen, lane);
            }
            // ---- stage C's candidates of this position
            const uint4 cw = S->cand[i];
            const uint32_t craw[4] = { cw.x, cw.y, cw.z, cw.w };
            uint32_t cl[4], cd[4];
#pragma unroll
            for (int t = 0; t < 4; t++) { cl[t] = LZP_CAND_LEN(craw[t]); if (cl[t] > maxLen) cl[t] = maxLen; cd[t] = LZP_CAND_DIST(craw[t]); }
            // ---- a long match ends the window: the path to here is committed and the match taken
            {
                uint32_t bl = 0, bd = 0; bool capped = false;
                if (rl0 > bl) { bl = rl0; bd = r0; }
                if (rl1 > bl) { bl = rl1; bd = r1; }
                if (rl2 > bl) { bl = rl2; bd = r2; }
                if (rl3 > bl) { bl = rl3; bd = r3; }
#pragma unroll
                for (int t = 0; t < 4; t++) if (cl[t] > bl) { bl = cl[t]; bd = cd[t]; capped = LZP_CAND_LEN(craw[t]) == LZP_CAND_LENCAP; }
                if (bl >= LZP_NICE) {
                    // a capped word says "at least 255": with no more than that left in the slice bl already is the length
                    longLen = (capped && maxLen > LZP_CAND_LENCAP) ? warp_extend(base, p - bd - 1u, p, 224u, maxLen, lane) : bl;
                    longDist = bd;
                    break;
                }
            }
            const uint32_t c0 = S->cost[i], room = W - i;
            const uint32_t pIsMatch = probs[LZM_ISMATCH + st * 16u + ps];
            const uint32_t pm0 = lzm_price(pt, pIsMatch, 0), pm1 = lzm_price(pt, pIsMatch, 1);
            // ---- literal: lanes 0..7 price one bit each (lane k = bit 7 - k, coded after the k bits above it)
            {
                const uint32_t sym = S->win[i + 1u], prev = S->win[i];
                const uint32_t mb = (st >= 7u) ? (uint32_t)__ldg(base + p - r0 - 1u) : 0u;
                uint32_t bitPrice = 0;
                if (lane < 8u) {
                    const uint32_t sh = 8u - lane, b = (sym >> (7u - lane)) & 1u;
                    const uint32_t m = (1u << lane) | (sym >> sh);
                    const bool matched = st >= 7u && (sym >> sh) == (mb >> sh);
                    const uint16_t* lp = probs + lzm_lit_base(q, p, prev);
                    const uint32_t mbit = (mb >> (7u - lane)) & 1u;
                    bitPrice = lzm_price(pt, matched ? lp[((1u + mbit) << 8) + m] : lp[m], b);
                }
                bitPrice += __shfl_xor_sync(B2Z_FULL, bitPrice, 1); bitPrice += __shfl_xor_sync(B2Z_FULL, bitPrice, 2); bitPrice += __shfl_xor_sync(B2Z_FULL, bitPrice, 4);
                const uint32_t cst = c0 + pm0 + __shfl_sync(B2Z_FULL, bitPrice, 0);
                if (lane == 0) {
                    S->litMb[i] = (uint8_t)mb;
                    if (cst < S->cost[i + 1u]) { S->cost[i + 1u] = cst; S->link[i + 1u] = PLINK(i, 1u, PK_LIT, 0u); }
                }
                if (end < i + 1u) end = i + 1u;
            }
            // ---- reps and matches: lane = length - 2 (all lengths are < LZP_NICE = 32 here); a lane owns target node i + length
            const uint32_t l = lane + 2u, tgt = i + l;
            const uint32_t pIsRep = probs[LZM_ISREP + st];
            const uint32_t prep = pm1 + lzm_price(pt, pIsRep, 1), pmatch = pm1 + lzm_price(pt, pIsRep, 0);
            {
                const uint32_t L0 = rl0 < room ? rl0 : room, L1 = rl1 < room ? rl1 : room, L2 = rl2 < room ? rl2 : room, L3 = rl3 < room ? rl3 : room;
                const uint32_t Lmax = max(max(L0, L1), max(L2, L3));
                if (Lmax >= 2u) {
                    const uint32_t lenP = (l <= Lmax) ? lzm_price_len(pt, probs + LZM_REPLEN, l, ps) : 0u;
                    const uint32_t g0 = probs[LZM_ISREPG0 + st], g1 = probs[LZM_ISREPG1 + st], g2 = probs[LZM_ISREPG2 + st];
                    if (L0 >= 2u) {
                        const uint32_t cst = c0 + prep + lzm_price(pt, g0, 0) + lzm_price(pt, probs[LZM_ISREP0LONG + st * 16u + ps], 1) + lenP;
                        if (l <= L0 && cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = PLINK(i, l, PK_REP, 0u); }
                    }
                    if (L1 >= 2u) {
                        const uint32_t cst = c0 + prep + lzm_price(pt, g0, 1) + lzm_price(pt, g1, 0) + lenP;
                        if (l <= L1 && cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = PLINK(i, l, PK_REP, 1u); }
                    }
                    if (L2 >= 2u) {
                        const uint32_t cst = c0 + prep + lzm_price(pt, g0, 1) + lzm_price(pt, g1, 1) + lzm_price(pt, g2, 0) + lenP;
                        if (l <= L2 && cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = PLINK(i, l, PK_REP, 2u); }
                    }
                    if (L3 >= 2u) {
                        const uint32_t cst = c0 + prep + lzm_price(pt, g0, 1) + lzm_price(pt, g1, 1) + lzm_price(pt, g2, 1) + lenP;
                        if (l <= L3 && cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = PLINK(i, l, PK_REP, 3u); }
                    }
                    if (end < i + Lmax) end = i + Lmax;
                }
            }
            {
                uint32_t ML = max(max(cl[0], cl[1]), max(cl[2], cl[3]));
                if (ML > room) ML = room;
                if (ML >= 2u) {
                    if (l <= ML) {                                   // every length goes with the nearest candidate that reaches it
                        uint32_t d = 0xFFFFFFFFu;
#pragma unroll
                        for (int t = 0; t < 4; t++) if (cl[t] >= l && cd[t] < d) d = cd[t];
                        const bool isRep = (rl0 && d == r0) || (rl1 && d == r1) || (rl2 && d == r2) || (rl3 && d == r3);   // stage R codes it as a rep: priced above
                        if (!isRep) {
                            const uint32_t cst = c0 + pmatch + lzm_price_len(pt, probs + LZM_LEN, l, ps) + lzm_price_dist(pt, probs, d, l - 2u < 4u ? l - 2u : 3u);
                            if (cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = PLINK(i, l, PK_MATCH, 0u); S->dist[tgt] = d; }
                        }
                    }
                    if (end < i + ML) end = i + ML;
                }
            }
            __syncwarp();                                            // node i + 1's arrival is complete and visible
            i++;
        }
        __syncwarp();
        // ---- commit the cheapest path to node i: its packets update the model as stage R will when it codes them
        if (lane == 0) {
            lzm_ctx x; x.state = S->ctx[0]; x.rep[0] = S->ctx[1]; x.rep[1] = S->ctx[2]; x.rep[2] = S->ctx[3]; x.rep[3] = S->ctx[4];
            uint32_t np = 0;
            for (uint32_t j = i; j > 0u; j = PLINK_FROM(S->link[j])) S->path[np++] = (uint16_t)j;
            while (np--) {
                const uint32_t j = S->path[np], lk = S->link[j], fr = PLINK_FROM(lk), kind = PLINK_KIND(lk), p = pos + fr;
                if (kind == PK_LIT) lzm_commit_literal_p(probs, &x, q, p, S->win[fr], S->win[fr + 1u], S->litMb[fr]);
                else {
                    const uint32_t d = kind == PK_MATCH ? S->dist[j] : x.rep[PLINK_R(lk)], len = PLINK_LEN(lk);
                    lzm_commit_match_p(probs, &x, q, p, len, d);
                    sink(p, len, d);
                }
            }
            if (longLen) { lzm_commit_match_p(probs, &x, q, pos + i, longLen, longDist); sink(pos + i, longLen, longDist); }
            S->ctx[0] = x.state; S->ctx[1] = x.rep[0]; S->ctx[2] = x.rep[1]; S->ctx[3] = x.rep[2]; S->ctx[4] = x.rep[3];
        }
        __syncwarp();
        pos += i + longLen;
    }
    if (lane == 0) fnseq[curBlk] = cnt;
}

#ifndef B2Z_CUEMU
size_t lzma2_cand_table_bytes(const EncGeom& g, uint32_t nWarps) { return (size_t)lzma2_cand_table_words(g.frameLog) * 4u * nWarps; }

void launch_lzma2_cand(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t* tables, uint32_t nWarps, uint32_t* cand, cudaStream_t st) {
    if (!srcSize) return;
    const uint32_t nFrames = (uint32_t)((srcSize + (1ull << g.frameLog) - 1) >> g.frameLog);
    lzma2_cand_kernel<<<nWarps < nFrames ? nWarps : nFrames, 32, 0, st>>>(src, srcSize, g, tables, cand);
}

cudaError_t launch_lzma2_parse(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint32_t* cand, uint64_t* seqs, uint32_t* nseq, cudaStream_t st) {
    if (!srcSize) return cudaSuccess;
    const uint64_t F = 1ull << g.frameLog;
    const uint32_t nFrames = (uint32_t)((srcSize + F - 1) >> g.frameLog);
    // counters of the blocks that exist: whole frames of F / 128 KiB blocks, then the last frame's
    const uint64_t lastBytes = srcSize - (uint64_t)(nFrames - 1u) * F;
    const size_t nBlocks = (size_t)(nFrames - 1u) * (size_t)(F >> 17) + (size_t)((lastBytes + B2Z_BLOCK - 1u) / B2Z_BLOCK);
    cudaError_t e = cudaMemsetAsync(nseq, 0, nBlocks * sizeof(uint32_t), st);
    if (e != cudaSuccess) return e;
    const size_t smem = lzma2_parse_smem_bytes(g.flags);
    const uint32_t nChains = nFrames * lzma2_enc_slices_per_frame(g);
    if (g.flags & B2Z_FLAG_LZ2_PROPS) {                             // lc / lp / pb other than the defaults: the run-time instantiation
        e = cudaFuncSetAttribute(lzma2_parse_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        lzma2_parse_kernel<true><<<nChains, 32, smem, st>>>(src, srcSize, g, cand, seqs, nseq, nChains);
    } else {
        e = cudaFuncSetAttribute(lzma2_parse_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        lzma2_parse_kernel<false><<<nChains, 32, smem, st>>>(src, srcSize, g, cand, seqs, nseq, nChains);
    }
    return cudaGetLastError();
}
#endif

}  // namespace b2z
