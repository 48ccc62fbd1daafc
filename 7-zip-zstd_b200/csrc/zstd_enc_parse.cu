// zstd_enc_parse.cu -- stage Z: the price-based parse of the block-parallel Zstandard encoder (flag B2Z_FLAG_ZSTD_OPT) for sm_90a.
//
// Replaces stage M for the high levels: stage C (lzma2_parse.cu: nearest-occurrence candidates by 3/4/6/8-byte keys, shared with
// method 21) runs first, then this kernel, one WARP per 128 KiB BLOCK -- blocks never share repcode history or entropy tables in
// this encoder (DESIGN.md 2.1), so a block is an independent chain, 32 768 of them per 4 GiB.
//
//   per block   byte histogram -> static literal prices; adaptive counts of the offset / match-length / literal-length codes
//               the block has produced so far -> sequence prices (b2z_zstd_cost.h)
//   per window  a forward dynamic programme over <= LZP_WIN positions in shared memory: node i = cheapest known coding of the
//               window's first i bytes + the state it leaves (repcode history, literals since the last match).  Lanes price a
//               node's edges in parallel: lane 0 the literal, lane l - 3 the repcode and candidate matches of length l (every
//               length goes with the nearest candidate that reaches it); a lane owns target node i + l.  A window ends where
//               all paths meet, at LZP_WIN nodes, or at a match of >= LZP_NICE bytes, which is taken at once.
//   commit      lane 0 walks the cheapest path: sequences (offBase with the repcode rules, literal run, length) go to the
//               block's array, counts are updated; the lanes then compact the path's literal bytes into the block's literals.
//
// Role in the reference: zstd_opt.c:1077 (ZSTD_compressBlock_opt_generic, levels 16-22), :590 (ZSTD_insertBtAndGetAllMatches),
// :295-356 (prices).  Output arrays = stage M's (what stage E reads).  Oracle statement: oracle/zstd_opt_oracle.c (identical).
#include "b2z_device.cuh"
#include "b2z_kernels.h"
#include "b2z_lzma_model.h"      // LZP_*: stage C's word layout, window size, nice length
#include "b2z_zstd_cost.h"

namespace b2z {

#define ZLINK(from, len, kind) ((from) | ((len) << 9) | ((kind) << 18))
#define ZLINK_FROM(x) ((x) & 0x1FFu)
#define ZLINK_LEN(x)  (((x) >> 9) & 0x1FFu)
#define ZLINK_KIND(x) (((x) >> 18) & 1u)

__constant__ zop_tables c_zop_tables = ZOP_TABLES_INIT;

struct ZParseSmem {                      // one warp's working set
    uint32_t cost[LZP_WIN + 1];
    uint32_t link[LZP_WIN + 1];          // best arrival: ZLINK(from, len, kind): kind 0 literal, 1 match
    uint32_t off[LZP_WIN + 1];           // ... its distance (matches)
    uint32_t rep[LZP_WIN + 1][3];        // state the best arrival leaves
    uint32_t litLen[LZP_WIN + 1];
    uint4    cand[LZP_WIN];
    uint32_t hist[256];
    zop_stats st;
    zop_tables tab;
    uint16_t litPrice[256];
    uint16_t path[LZP_WIN + 1];
    uint8_t  isLit[LZP_WIN + 8];
    uint8_t  win[LZP_WIN + 40];          // win[k] = frame byte pos + k
    uint32_t ctx[4];                     // committed state: rep0..2, litLen
    uint32_t counters[2];                // nseq, nlit of the block so far
};
size_t zstd_enc_parse_smem_bytes() { return sizeof(ZParseSmem); }

__global__ void __launch_bounds__(32)
zstd_enc_parse_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, const uint32_t* __restrict__ cand,
                      uint64_t* __restrict__ seqs, uint32_t* __restrict__ nseq, uint8_t* __restrict__ lits, uint32_t* __restrict__ nlit, uint32_t nBlocksTotal) {
    B2Z_DYN_SMEM(ZParseSmem, S);
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t gb = blockIdx.x;                                 // block index: frame * blocksPerFrame + block
    if (gb >= nBlocksTotal) return;
    const uint64_t F = 1ull << g.frameLog;
    const uint32_t bpf = (uint32_t)(F >> 17);
    const uint32_t f = gb / bpf, blk = gb - f * bpf;
    const uint64_t f0 = (uint64_t)f << g.frameLog;
    const uint32_t n = (uint32_t)((srcSize - f0) < F ? (srcSize - f0) : F);
    const uint32_t b0 = blk * B2Z_BLOCK;
    if (b0 >= n) return;                                            // block beyond the end of a short last frame
    const uint32_t b1 = (b0 + B2Z_BLOCK) < n ? (b0 + B2Z_BLOCK) : n;
    const uint8_t* __restrict__ base = src + f0;
    const uint4* __restrict__ cand4 = reinterpret_cast<const uint4*>(cand) + f0;
    uint64_t* const bseqs = seqs + (size_t)gb * B2Z_MAXSEQ;
    uint8_t* const blits = lits + f0 + b0;
    const zop_tables* const tab = &S->tab;
    zop_stats* const st = &S->st;

    // ---- per block: tables, byte histogram -> literal prices, fresh counts and state
    {
        const uint8_t* ct = reinterpret_cast<const uint8_t*>(&c_zop_tables);
        uint8_t* dt = reinterpret_cast<uint8_t*>(&S->tab);
        for (uint32_t k = lane; k < (uint32_t)sizeof(zop_tables); k += 32u) dt[k] = ct[k];
        for (uint32_t k = lane; k < 256u; k += 32u) S->hist[k] = 0;
        for (uint32_t k = lane; k < ZOP_N_OF; k += 32u) st->of[k] = 1;
        for (uint32_t k = lane; k < ZOP_N_ML; k += 32u) st->ml[k] = 1;
        for (uint32_t k = lane; k < ZOP_N_LL; k += 32u) st->ll[k] = 1;
        if (lane == 0) { st->ofSum = ZOP_N_OF; st->mlSum = ZOP_N_ML; st->llSum = ZOP_N_LL; S->ctx[0] = S->ctx[1] = S->ctx[2] = S->ctx[3] = 0; S->counters[0] = S->counters[1] = 0; }
        __syncwarp();
        for (uint32_t p = b0 + lane; p < b1; p += 32u) atomicAdd(&S->hist[__ldg(base + p)], 1u);
        __syncwarp();
        for (uint32_t k = lane; k < 256u; k += 32u) { const uint32_t h = S->hist[k]; S->litPrice[k] = (uint16_t)(h ? zop_cost(tab, h, b1 - b0) : 0u); }
        __syncwarp();
    }

    uint32_t pos = b0;
    while (pos < b1) {
        const uint32_t W = (b1 - pos) < LZP_WIN ? (b1 - pos) : LZP_WIN;
        for (uint32_t k = lane; k < W + 32u; k += 32u) S->win[k] = (pos + k < b1) ? __ldg(base + pos + k) : (uint8_t)0;
        for (uint32_t k = lane; k < W; k += 32u) { S->cand[k] = __ldg(cand4 + pos + k); S->isLit[k] = 0; }
        for (uint32_t k = lane; k <= W; k += 32u) S->cost[k] = k ? 0xFFFFFFFFu : 0u;
        if (lane == 0) { S->rep[0][0] = S->ctx[0]; S->rep[0][1] = S->ctx[1]; S->rep[0][2] = S->ctx[2]; S->litLen[0] = S->ctx[3]; }
        __syncwarp();

        uint32_t end = 0, i = 0, longLen = 0, longOff = 0;
        zop_ctx cx; cx.rep[0] = S->ctx[0]; cx.rep[1] = S->ctx[1]; cx.rep[2] = S->ctx[2]; cx.litLen = S->ctx[3];      // state of node i (warp-uniform)
        for (;;) {
            if (i) {                                                // node i is final: the state its best arrival leaves
                const uint32_t lk = S->link[i], fr = ZLINK_FROM(lk);
                cx.rep[0] = S->rep[fr][0]; cx.rep[1] = S->rep[fr][1]; cx.rep[2] = S->rep[fr][2]; cx.litLen = S->litLen[fr];
                if (ZLINK_KIND(lk) == 0u) cx.litLen += 1u; else zop_after_match(&cx, S->off[i]);
                if (lane == 0) { S->rep[i][0] = cx.rep[0]; S->rep[i][1] = cx.rep[1]; S->rep[i][2] = cx.rep[2]; S->litLen[i] = cx.litLen; }
            }
            if (i == W || (i && i == end)) break;
            const uint32_t p = pos + i, maxLen = b1 - p, room = W - i;
            const uint32_t lim32 = maxLen < 32u ? maxLen : 32u;
            const uint32_t curB = S->win[i + lane];
            // ---- repcode offsets as the next sequence would see them (shifted when no literal precedes it) and their lengths
            uint32_t o0, o1, o2;
            if (cx.litLen) { o0 = cx.rep[0]; o1 = cx.rep[1]; o2 = cx.rep[2]; }
            else { o0 = cx.rep[1]; o1 = cx.rep[2]; o2 = cx.rep[0] > 1u ? cx.rep[0] - 1u : 0u; }
            uint32_t rl0, rl1, rl2;
            {
                const bool v0 = o0 && p >= o0, v1 = o1 && o1 != o0 && p >= o1, v2 = o2 && o2 != o0 && o2 != o1 && p >= o2;
                const uint32_t x0 = (v0 && lane < lim32) ? (uint32_t)__ldg(base + p - o0 + lane) : 256u;
                const uint32_t x1 = (v1 && lane < lim32) ? (uint32_t)__ldg(base + p - o1 + lane) : 256u;
                const uint32_t x2 = (v2 && lane < lim32) ? (uint32_t)__ldg(base + p - o2 + lane) : 256u;
                const uint32_t m0 = __ballot_sync(B2Z_FULL, x0 != curB), m1 = __ballot_sync(B2Z_FULL, x1 != curB), m2 = __ballot_sync(B2Z_FULL, x2 != curB);
                rl0 = m0 ? (uint32_t)(__ffs((int)m0) - 1) : 32u; rl1 = m1 ? (uint32_t)(__ffs((int)m1) - 1) : 32u; rl2 = m2 ? (uint32_t)(__ffs((int)m2) - 1) : 32u;
                if (rl0 == 32u && maxLen > 32u) rl0 = warp_extend(base, p - o0, p, 32u, maxLen, lane);
                if (rl1 == 32u && maxLen > 32u) rl1 = warp_extend(base, p - o1, p, 32u, maxLen, lane);
                if (rl2 == 32u && maxLen > 32u) rl2 = warp_extend(base, p - o2, p, 32u, maxLen, lane);
            }
            // ---- stage C's candidates of this position
            const uint4 cw = S->cand[i];
            const uint32_t craw[4] = { cw.x, cw.y, cw.z, cw.w };
            uint32_t cl[4], co[4];
#pragma unroll
            for (int t = 0; t < 4; t++) { cl[t] = LZP_CAND_LEN(craw[t]); if (cl[t] > maxLen) cl[t] = maxLen; co[t] = LZP_CAND_DIST(craw[t]) + 1u; }
            // ---- a long match ends the window: the path to here is committed and the match taken
            {
                uint32_t bl = 0, bo = 0; bool capped = false;
                if (rl0 > bl) { bl = rl0; bo = o0; }
                if (rl1 > bl) { bl = rl1; bo = o1; }
                if (rl2 > bl) { bl = rl2; bo = o2; }
#pragma unroll
                for (int t = 0; t < 4; t++) if (cl[t] > bl) { bl = cl[t]; bo = co[t]; capped = LZP_CAND_LEN(craw[t]) == LZP_CAND_LENCAP; }
                if (bl >= LZP_NICE) {
                    // a capped word says "at least 255": with no more than that left in the block bl already is the length
                    longLen = (capped && maxLen > LZP_CAND_LENCAP) ? warp_extend(base, p - bo, p, 224u, maxLen, lane) : bl;
                    longOff = bo;
                    break;
                }
            }
            const uint32_t c0 = S->cost[i];
            if (lane == 0) {                                        // literal
                const uint32_t cst = c0 + S->litPrice[S->win[i]];
                if (cst < S->cost[i + 1u]) { S->cost[i + 1u] = cst; S->link[i + 1u] = ZLINK(i, 1u, 0u); }
            }
            if (end < i + 1u) end = i + 1u;
            // ---- repcode and candidate matches: lane = length - 3 (all lengths are < LZP_NICE here); a lane owns target node i + length
            const uint32_t l = lane + ZOP_MINMATCH, tgt = i + l;
            const uint32_t L0 = rl0 < room ? rl0 : room, L1 = rl1 < room ? rl1 : room, L2 = rl2 < room ? rl2 : room;
            uint32_t ML = max(max(cl[0], cl[1]), max(cl[2], cl[3]));
            if (ML > room) ML = room;
            const uint32_t Lany = max(max(L0, L1), max(L2, ML));
            if (Lany >= ZOP_MINMATCH) {
                // price of a sequence = literal-run part (same for all edges of this node) + offset part + length part (per lane)
                const uint32_t lc = zop_ll_code(tab, cx.litLen);
                const uint32_t llP = 16u * tab->llBits[lc] + zop_cost(tab, st->ll[lc], st->llSum);
                uint32_t mlP = 0;
                if (l <= Lany) { const uint32_t mc = zop_ml_code(tab, l - ZOP_MINMATCH); mlP = 16u * tab->mlBits[mc] + zop_cost(tab, st->ml[mc], st->mlSum); }
                if (L0 >= ZOP_MINMATCH) {
                    const uint32_t oc = zop_highbit(zop_off_base(&cx, o0));
                    const uint32_t cst = c0 + llP + 16u * oc + zop_cost(tab, st->of[oc], st->ofSum) + mlP;
                    if (l <= L0 && cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = ZLINK(i, l, 1u); S->off[tgt] = o0; }
                    if (end < i + L0) end = i + L0;
                }
                if (L1 >= ZOP_MINMATCH) {
                    const uint32_t oc = zop_highbit(zop_off_base(&cx, o1));
                    const uint32_t cst = c0 + llP + 16u * oc + zop_cost(tab, st->of[oc], st->ofSum) + mlP;
                    if (l <= L1 && cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = ZLINK(i, l, 1u); S->off[tgt] = o1; }
                    if (end < i + L1) end = i + L1;
                }
                if (L2 >= ZOP_MINMATCH) {
                    const uint32_t oc = zop_highbit(zop_off_base(&cx, o2));
                    const uint32_t cst = c0 + llP + 16u * oc + zop_cost(tab, st->of[oc], st->ofSum) + mlP;
                    if (l <= L2 && cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = ZLINK(i, l, 1u); S->off[tgt] = o2; }
                    if (end < i + L2) end = i + L2;
                }
                if (ML >= ZOP_MINMATCH) {
                    if (l <= ML) {                                  // every length goes with the nearest candidate that reaches it
                        uint32_t o = 0xFFFFFFFFu;
#pragma unroll
                        for (int t = 0; t < 4; t++) if (cl[t] >= l && co[t] < o) o = co[t];
                        const uint32_t oc = zop_highbit(zop_off_base(&cx, o));
                        const uint32_t cst = c0 + llP + 16u * oc + zop_cost(tab, st->of[oc], st->ofSum) + mlP;
                        if (cst < S->cost[tgt]) { S->cost[tgt] = cst; S->link[tgt] = ZLINK(i, l, 1u); S->off[tgt] = o; }
                    }
                    if (end < i + ML) end = i + ML;
                }
            }
            __syncwarp();                                           // node i + 1's arrival is complete and visible
            i++;
        }
        __syncwarp();
        // ---- commit the cheapest path to node i
        if (lane == 0) {
            zop_ctx x; x.rep[0] = S->ctx[0]; x.rep[1] = S->ctx[1]; x.rep[2] = S->ctx[2]; x.litLen = S->ctx[3];
            uint32_t ns = S->counters[0];
            uint32_t np = 0;
            for (uint32_t j = i; j > 0u; j = ZLINK_FROM(S->link[j])) S->path[np++] = (uint16_t)j;
            while (np--) {
                const uint32_t j = S->path[np], lk = S->link[j], fr = ZLINK_FROM(lk);
                if (ZLINK_KIND(lk) == 0u) { S->isLit[fr] = 1; x.litLen++; continue; }
                const uint32_t len = ZLINK_LEN(lk), off = S->off[j];
                if (ns >= B2Z_MAXSEQ) { for (uint32_t k = 0; k < len; k++) S->isLit[fr + k] = 1; x.litLen += len; continue; }   // array full: the bytes stay literals
                const uint32_t ob = zop_off_base(&x, off);
                zop_count_seq(tab, st, x.litLen, ob, len);
                bseqs[ns++] = B2Z_PACK_SEQ(ob, x.litLen, len);
                zop_after_match(&x, off);
            }
            S->counters[0] = ns;
            S->ctx[0] = x.rep[0]; S->ctx[1] = x.rep[1]; S->ctx[2] = x.rep[2]; S->ctx[3] = x.litLen;
        }
        __syncwarp();
        // ---- the path's literal bytes, compacted in position order
        {
            uint32_t nl = S->counters[1];
            for (uint32_t k0 = 0; k0 < i; k0 += 32u) {
                const uint32_t k = k0 + lane;
                const bool isl = k < i && S->isLit[k];
                const uint32_t m = __ballot_sync(B2Z_FULL, isl);
                if (isl) blits[nl + (uint32_t)__popc(m & ((1u << lane) - 1u))] = S->win[k];
                nl += (uint32_t)__popc(m);
            }
            if (lane == 0) S->counters[1] = nl;
            __syncwarp();
        }
        pos += i;
        // ---- the long match, if one ended the window
        if (longLen) {
            const uint32_t ns = S->counters[0];
            if (ns >= B2Z_MAXSEQ) {                                 // array full: its bytes stay literals
                const uint32_t nl = S->counters[1];
                for (uint32_t k = lane; k < longLen; k += 32u) blits[nl + k] = __ldg(base + pos + k);
                __syncwarp();
                if (lane == 0) { S->counters[1] = nl + longLen; S->ctx[3] += longLen; }
            } else if (lane == 0) {
                zop_ctx x; x.rep[0] = S->ctx[0]; x.rep[1] = S->ctx[1]; x.rep[2] = S->ctx[2]; x.litLen = S->ctx[3];
                const uint32_t ob = zop_off_base(&x, longOff);
                zop_count_seq(tab, st, x.litLen, ob, longLen);
                bseqs[ns] = B2Z_PACK_SEQ(ob, x.litLen, longLen);
                zop_after_match(&x, longOff);
                S->counters[0] = ns + 1u;
                S->ctx[0] = x.rep[0]; S->ctx[1] = x.rep[1]; S->ctx[2] = x.rep[2]; S->ctx[3] = x.litLen;
            }
            pos += longLen;
        }
        __syncwarp();
    }
    if (lane == 0) { nseq[gb] = S->counters[0]; nlit[gb] = S->counters[1]; }
}

#ifndef B2Z_CUEMU
// stage Z for the frames of src (dense frames only); cand = stage C's words
cudaError_t launch_zstd_enc_parse(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint32_t* cand,
                                  uint64_t* seqs, uint32_t* nseq, uint8_t* lits, uint32_t* nlit, cudaStream_t st) {
    if (!srcSize) return cudaSuccess;
    const uint64_t F = 1ull << g.frameLog;
    const uint32_t nFrames = (uint32_t)((srcSize + F - 1) >> g.frameLog);
    const uint64_t lastBytes = srcSize - (uint64_t)(nFrames - 1u) * F;
    const uint32_t nBlocks = (nFrames - 1u) * (uint32_t)(F >> 17) + (uint32_t)((lastBytes + B2Z_BLOCK - 1u) / B2Z_BLOCK);
    cudaError_t e = cudaFuncSetAttribute(zstd_enc_parse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ZParseSmem));
    if (e != cudaSuccess) return e;
    zstd_enc_parse_kernel<<<nBlocks, 32, sizeof(ZParseSmem), st>>>(src, srcSize, g, cand, seqs, nseq, lits, nlit, nBlocks);
    return cudaGetLastError();
}
#endif

}  // namespace b2z
