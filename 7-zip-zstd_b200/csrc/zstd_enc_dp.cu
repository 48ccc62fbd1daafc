// zstd_enc_dp.cu -- stage G of the block-parallel Zstandard encoder (sm_90a): the parse.
//
// One WARP owns one 128 KiB block, one LANE one 4 KiB segment of it (B2Z_SEG): 32 768 blocks x 32 lanes per 4 GiB, so the
// strictly sequential part of the parse -- a minimum-price path -- runs as a million independent chains.  Per block:
//   1. literal prices: byte histogram of the first 64 of every 256 bytes (coalesced 16-byte loads, shared-memory atomics),
//      price = log2(total / count) in 1/16 bit, clamped;
//   2. per lane, a backward dynamic programme over its segment: cost[i] = min(literal + cost[i+1], the position's
//      candidate (stage F) at its length L, L-1, L-2: B2Z_DP_MATCH + offset extra bits + cost[i+l]).  Only the
//      next B2Z_CAP costs are live (candidates are at most B2Z_CAP long), kept in a per-lane ring in shared memory; the choice
//      (0 = literal, else the length) goes to a byte array in HBM, four positions per store;
//   3. per lane, a forward walk that only counts (sequences, literals, where the last match ends) -- a chosen match of
//      the full B2Z_CAP bytes is extended by direct comparison to the segment end;
//   4. warp scans turn the counts into each lane's place in the block's sequence and literal arrays and into the literal
//      run that reaches into a lane from the lanes before it;
//   5. the same walk again, emitting final (offBase, litLength, matchLength) records and the literal bytes.  The repcode
//      history is "unknown" at every segment start, so no lane waits for another.
// A block of one repeated byte becomes the single sequence that stage E stores as an RLE block.
//
// Role in the reference: the parse half of ZSTD_compressBlock_doubleFast_noDict_generic (zstd_double_fast.c:103-330: which
// match to take, ZSTD_storeSeq, ZSTD_updateRep zstd_compress_internal.h:775,817) -- done here by price, which is what pays
// for stage F's small tables.  Sequential statement: oracle/zstd_enc_oracle.c:parse_frame; outputs must be identical.
#include "b2z_device.cuh"
#include "b2z_kernels.h"
#include "b2z_zstd_cost.h"

namespace b2z {

// Memory access: a lane's segment lies 4 KiB (16 KiB of candidate words) away from its neighbour's, so lanes never read HBM
// themselves.  The warp moves TILES of 32 positions per lane through shared memory instead: row j of a tile = the 32
// positions lane j works on next, loaded / stored by the whole warp as 128-byte (candidates) or 32-byte (input bytes,
// choices) coalesced pieces, read by lane j along its padded row (stride 33 / 9 words: conflict-free).
constexpr uint32_t DP_RING = 32;
static_assert(DP_RING > B2Z_CAP && (DP_RING & (DP_RING - 1u)) == 0, "the ring holds cost[i + 1 .. i + B2Z_CAP] while cost[i] is written");
struct DpWarpSmem {
    uint32_t ring[DP_RING][32];  // cost ring: [position & (DP_RING - 1)][lane]; a candidate reaches at most B2Z_CAP positions ahead
    uint32_t candTile[32][33];   // [lane][position in tile]; the byte histogram (256 words) lives here before the first tile
    uint32_t srcTile[32][9];     // [lane][4 input bytes]
    uint32_t chcTile[32][9];     // [lane][4 choices]
    uint8_t litc[256];
};

// 16 * log2(x) as b2z_zstd_cost.h:zop_log16, with the fraction table in registers
__device__ __forceinline__ uint32_t dp_log16(uint32_t x) {
    const uint32_t hb = highbit32(x);
    const uint32_t k = hb >= 4u ? ((x >> (hb - 4u)) & 15u) : ((x << (4u - hb)) & 15u);
    // ZOP_FRAC_LIST (1,2,3,5,6,7,8,9 | 10,11,12,13,14,15,15,16) as two words of bytes
    const uint64_t lo = 0x0908070605030201ull, hi = 0x100F0F0E0D0C0B0Aull;
    const uint32_t fr = (uint32_t)(((k < 8u ? lo : hi) >> ((k & 7u) * 8u)) & 0xFFu);
    return 16u * hb + ((k == 0u && (x & (x - 1u)) == 0u) ? 0u : fr);
}

// tile t of a 32-bit-per-position array: 32 coalesced 128-byte rows.  base = the block's array, bn = positions in the block
__device__ __forceinline__ void dp_load_cand_tile(DpWarpSmem& sm, const uint32_t* __restrict__ base, uint32_t bn, uint32_t t, uint32_t lane) {
#pragma unroll 8
    for (uint32_t j = 0; j < 32u; j++) {
        const uint32_t pos = j * B2Z_SEG + 32u * t + lane;
        sm.candTile[j][lane] = pos < bn ? __ldcs(base + pos) : 0u;
    }
}
// tile t of a byte-per-position array: 8 loads of 4 rows x 32 bytes
__device__ __forceinline__ void dp_load_byte_tile(uint32_t (*tile)[9], const uint8_t* __restrict__ base, uint32_t bn, uint32_t t, uint32_t lane) {
#pragma unroll
    for (uint32_t r = 0; r < 8u; r++) {
        const uint32_t row = 4u * r + (lane >> 3), wd = lane & 7u, pos = row * B2Z_SEG + 32u * t + 4u * wd;
        tile[row][wd] = pos < bn ? __ldg(reinterpret_cast<const uint32_t*>(base + pos)) : 0u;
    }
}
__device__ __forceinline__ void dp_store_byte_tile(const uint32_t (*tile)[9], uint8_t* __restrict__ base, uint32_t bn, uint32_t t, uint32_t lane) {
#pragma unroll
    for (uint32_t r = 0; r < 8u; r++) {
        const uint32_t row = 4u * r + (lane >> 3), wd = lane & 7u, pos = row * B2Z_SEG + 32u * t + 4u * wd;
        if (pos < bn) *reinterpret_cast<uint32_t*>(base + pos) = tile[row][wd];
    }
}

// per-lane state of the forward walk over a segment's choices
struct DpWalk {
    uint32_t i, ns, nl, lastEnd;            // segment-relative position; sequences / literals so far; block-relative end of the last match
    uint32_t rep0, rep1, rep2, prevEnd;     // EMIT only
};

// bit t of the result: byte t of the lane's 32-byte row is not zero (4 bytes per step: carry-free "byte != 0", then a multiply that
// gathers the four flag bits)
__device__ __forceinline__ uint32_t dp_nonzero_mask(const uint32_t* row) {
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t w = row[k];
        const uint32_t f = ((((w & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | w) & 0x80808080u) >> 7;     // bits 0, 8, 16, 24
        m |= ((f * 0x00204081u) >> 21 & 15u) << (4 * k);
    }
    return m;
}

// one tile of the forward walk: positions [32 t, 32 t + 32) of the lane's segment, as far as the lane's path touches them.  On the
// path, literals are exactly the positions up to the next non-zero choice, so a whole literal run is one iteration (find-first-set on
// the tile's "choice != 0" mask), and the loop runs once per match instead of once per position.
template <bool EMIT>
__device__ __forceinline__ void dp_walk_tile(DpWarpSmem& sm, DpWalk& k, uint32_t t, uint32_t lane, uint32_t sn, uint32_t s0 /* block-relative */,
                                             const uint64_t* __restrict__ fw /* frame as words */, uint32_t segAbs /* frame-relative */, uint32_t nWords,
                                             const uint32_t* __restrict__ cnd /* segment's candidate words */,
                                             uint64_t* __restrict__ outSeq, uint8_t* __restrict__ outLit) {
    const uint32_t tEnd = (32u * t + 32u) < sn ? (32u * t + 32u) : sn;
    if (k.i >= tEnd) return;
    const uint32_t inTile = tEnd - 32u * t;
    const uint32_t M = dp_nonzero_mask(sm.chcTile[lane]) & (inTile >= 32u ? 0xFFFFFFFFu : ((1u << inTile) - 1u));
    while (k.i < tEnd) {
        uint32_t w = k.i & 31u;
        const uint32_t rem = M >> w;
        const uint32_t r = rem ? (uint32_t)(__ffs((int)rem) - 1) : (tEnd - k.i);        // literals up to the next match of the tile (or the tile's end)
        if (r) {
            if (EMIT) for (uint32_t j = 0; j < r; j++) { const uint32_t ww = w + j; outLit[k.nl + j] = (uint8_t)(sm.srcTile[lane][ww >> 2] >> (8u * (ww & 3u))); }
            k.nl += r; k.i += r; w += r;
            if (!rem) break;
        }
        uint32_t l = (sm.chcTile[lane][w >> 2] >> (8u * (w & 3u))) & 255u;
        const uint32_t off = EMIT ? B2Z_CAND_OFF(sm.candTile[lane][w]) : 0u;
        if (l == B2Z_CAP) {                                                    // the full common prefix, to the segment end at most
            const uint32_t o = EMIT ? off : B2Z_CAND_OFF(__ldg(cnd + k.i));
            l = match_len(fw, segAbs + k.i - o, segAbs + k.i, sn - k.i, nWords);
        }
        if (EMIT) {
            const uint32_t pos = s0 + k.i, ll = pos - k.prevEnd;
            uint32_t code = 0, offBase;
            if (ll) { if (off == k.rep0) code = 1; else if (off == k.rep1) code = 2; else if (off == k.rep2) code = 3; }
            else { if (off == k.rep1) code = 1; else if (off == k.rep2) code = 2; else if (k.rep0 > 1u && off == k.rep0 - 1u) code = 3; }
            if (code == 0) { offBase = off + 3u; k.rep2 = k.rep1; k.rep1 = k.rep0; k.rep0 = off; }
            else {
                offBase = code;
                const uint32_t idx = code - 1u + (ll == 0u);
                if (idx != 0) {
                    const uint32_t cur = idx == 3 ? k.rep0 - 1u : (idx == 1 ? k.rep1 : k.rep2);
                    if (idx != 1) k.rep2 = k.rep1;
                    k.rep1 = k.rep0; k.rep0 = cur;
                }
            }
            outSeq[k.ns] = B2Z_PACK_SEQ(offBase, ll, l);
            k.prevEnd = pos + l;
        }
        k.ns++; k.i += l; k.lastEnd = s0 + k.i;
    }
}

__global__ void __launch_bounds__(B2Z_DP_WARPS * 32)
zstd_enc_dp_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, const uint32_t* __restrict__ cand, uint8_t* __restrict__ choice,
                   uint64_t* __restrict__ seqs, uint32_t* __restrict__ nseq, uint8_t* __restrict__ lits, uint32_t* __restrict__ nlit,
                   uint32_t nBlockSlots) {
    B2Z_DYN_SMEM(DpWarpSmem, allSm);
    const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
    DpWarpSmem& sm = allSm[wib];
    const uint32_t bw = blockIdx.x * B2Z_DP_WARPS + wib;                       // block slot: frame * blocksPerFrame + block in frame
    if (bw >= nBlockSlots) return;
    const uint32_t bpf = 1u << (g.frameLog - 17u);
    const uint64_t f = bw >> (g.frameLog - 17u);
    const uint32_t b = bw & (bpf - 1u);
    const uint32_t n = enc_frame_bytes(g, srcSize, f);
    const uint32_t b0 = b << 17;
    if (b0 >= n) return;                                                       // the last frame may hold fewer blocks
    const uint32_t bn = (n - b0) < B2Z_BLOCK ? (n - b0) : B2Z_BLOCK;
    const uint64_t f0 = f << g.frameLog;
    const uint8_t* __restrict__ fb = src + f0;
    const uint8_t* __restrict__ bs = fb + b0;
    const uint32_t* __restrict__ cndB = cand + f0 + b0;
    uint8_t* __restrict__ chcB = choice + f0 + b0;
    uint64_t* __restrict__ out = seqs + (size_t)bw * B2Z_MAXSEQ;
    uint8_t* __restrict__ lit = lits + f0 + b0;
    const uint32_t nTiles = ((bn < B2Z_SEG ? bn : B2Z_SEG) + 31u) >> 5;        // tiles of the longest segment (the first)

    // ---- 1. literal prices
    uint32_t* const hist = &sm.candTile[0][0];
    for (uint32_t i = lane; i < 256u; i += 32u) hist[i] = 0;
    __syncwarp();
    for (uint32_t idx = lane;; idx += 32u) {
        const uint32_t o = (idx >> 2) * 256u + (idx & 3u) * 16u;              // 4 lanes per sampled 64-byte run
        if ((idx & ~31u) * 64u >= bn) break;                                   // warp-uniform: the step's first run starts past the block
        if (o + 16u <= bn) {
            const uint4 q = __ldg(reinterpret_cast<const uint4*>(bs + o));
            const uint32_t ws[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
            for (int k = 0; k < 4; k++) { atomicAdd(&hist[ws[k] & 255u], 1u); atomicAdd(&hist[(ws[k] >> 8) & 255u], 1u); atomicAdd(&hist[(ws[k] >> 16) & 255u], 1u); atomicAdd(&hist[ws[k] >> 24], 1u); }
        } else for (uint32_t k = o; k < bn && k < o + 16u; k++) atomicAdd(&hist[bs[k]], 1u);
    }
    __syncwarp();
    {
        uint32_t part = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) part += hist[lane * 8u + k];
#pragma unroll
        for (int d = 16; d; d >>= 1) part += __shfl_xor_sync(B2Z_FULL, part, d);
        const uint32_t lt = dp_log16(part);
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const uint32_t h = hist[lane * 8u + k];
            uint32_t v = B2Z_DP_LIT_MAX;
            if (h) { const uint32_t lh = dp_log16(h); v = lt > lh ? lt - lh : 1u; }
            sm.litc[lane * 8u + k] = (uint8_t)(v < B2Z_DP_LIT_MIN ? B2Z_DP_LIT_MIN : (v > B2Z_DP_LIT_MAX ? B2Z_DP_LIT_MAX : v));
        }
    }
    __syncwarp();

    // ---- 2. backward dynamic programme, tile by tile from the segment's end
    const uint32_t s0 = lane * B2Z_SEG;
    const bool active = s0 < bn;
    const uint32_t sn = active ? ((bn - s0) < B2Z_SEG ? (bn - s0) : B2Z_SEG) : 0u;
    uint32_t diff = 0;                                                         // any byte of the segment unlike the block's first byte
    const uint32_t first = bs[0];
    if (active) sm.ring[sn & (DP_RING - 1u)][lane] = 0;
    for (uint32_t t = nTiles; t-- > 0;) {
        dp_load_cand_tile(sm, cndB, bn, t, lane);
        dp_load_byte_tile(sm.srcTile, bs, bn, t, lane);
        __syncwarp();
        if (32u * t < sn) {
            const bool full = 32u * t + 32u <= sn;                             // only the last tile of a short segment is not
#pragma unroll 2
            for (int wi = 7; wi >= 0; wi--) {
                const uint32_t b4 = sm.srcTile[lane][wi];
                uint32_t packed = 0;
#pragma unroll
                for (int j = 3; j >= 0; j--) {
                    const uint32_t i = 32u * t + 4u * (uint32_t)wi + (uint32_t)j;
                    if (!full && i >= sn) continue;
                    // branch-free: an absent or too short candidate prices at 2^31 and loses against the literal
                    const uint32_t byte = (b4 >> (8 * j)) & 255u;
                    diff |= byte ^ first;
                    const uint32_t c = sm.candTile[lane][4 * wi + j];
                    const uint32_t len = B2Z_CAND_LEN(c), ob = 16u * highbit32(B2Z_CAND_OFF(c) + 3u) + B2Z_DP_MATCH;
                    uint32_t best = (uint32_t)sm.litc[byte] + sm.ring[(i + 1u) & (DP_RING - 1u)][lane], ch = 0;
#pragma unroll
                    for (uint32_t k = 0; k <= B2Z_DP_NTRUNC; k++) {
                        const uint32_t l = len - k;                            // wraps below zero when len < k: the index stays inside the ring, the price is discarded
                        const uint32_t pr = ob + sm.ring[(i + l) & (DP_RING - 1u)][lane];
                        const bool take = (len >= B2Z_DP_MINLEN + k) && pr < best;
                        best = take ? pr : best; ch = take ? l : ch;
                    }
                    sm.ring[i & (DP_RING - 1u)][lane] = best;
                    packed |= ch << (8 * j);
                }
                sm.chcTile[lane][wi] = packed;
            }
        }
        __syncwarp();
        dp_store_byte_tile(sm.chcTile, chcB, bn, t, lane);
        __syncwarp();
    }
    // ---- one repeated byte: the canonical single sequence (stage E emits an RLE block for it)
    if (!__any_sync(B2Z_FULL, diff != 0u) && bn > 1u) {
        if (lane == 0) { out[0] = B2Z_PACK_SEQ(1u + 3u, 1u, bn - 1u); lit[0] = bs[0]; nseq[bw] = 1u; nlit[bw] = 1u; }
        return;
    }

    const uint64_t* __restrict__ fw = reinterpret_cast<const uint64_t*>(fb);
    const uint32_t nWords = (n + 7u) >> 3;
    const uint32_t* __restrict__ cnd = cndB + s0;
    // ---- 3. count
    DpWalk k; k.i = 0; k.ns = 0; k.nl = 0; k.lastEnd = 0; k.rep0 = k.rep1 = k.rep2 = 0; k.prevEnd = 0;
    for (uint32_t t = 0; t < nTiles; t++) {
        dp_load_byte_tile(sm.chcTile, chcB, bn, t, lane);
        __syncwarp();
        dp_walk_tile<false>(sm, k, t, lane, sn, s0, fw, b0 + s0, nWords, cnd, nullptr, nullptr);
        __syncwarp();
    }
    const uint32_t cntSeq = k.ns, cntLit = k.nl;
    // ---- 4. places: exclusive sums of the counts, exclusive maximum of the last match ends
    uint32_t seqBase = cntSeq, litBase = cntLit, prevEnd = cntSeq ? k.lastEnd : 0u;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t a = __shfl_up_sync(B2Z_FULL, seqBase, d), c = __shfl_up_sync(B2Z_FULL, litBase, d), e = __shfl_up_sync(B2Z_FULL, prevEnd, d);
        if (lane >= (uint32_t)d) { seqBase += a; litBase += c; prevEnd = e > prevEnd ? e : prevEnd; }
    }
    const uint32_t totSeq = __shfl_sync(B2Z_FULL, seqBase, 31), totLit = __shfl_sync(B2Z_FULL, litBase, 31);
    seqBase -= cntSeq; litBase -= cntLit;
    prevEnd = __shfl_up_sync(B2Z_FULL, prevEnd, 1); if (lane == 0) prevEnd = 0;
    // ---- 5. emit
    k.i = 0; k.ns = 0; k.nl = 0; k.prevEnd = prevEnd;
    for (uint32_t t = 0; t < nTiles; t++) {
        dp_load_byte_tile(sm.chcTile, chcB, bn, t, lane);
        dp_load_byte_tile(sm.srcTile, bs, bn, t, lane);
        dp_load_cand_tile(sm, cndB, bn, t, lane);
        __syncwarp();
        dp_walk_tile<true>(sm, k, t, lane, sn, s0, fw, b0 + s0, nWords, cnd, out + seqBase, lit + litBase);
        __syncwarp();
    }
    if (lane == 0) { nseq[bw] = totSeq; nlit[bw] = totLit; }
}

#ifndef B2Z_CUEMU
size_t zstd_enc_dp_smem_bytes() { return sizeof(DpWarpSmem) * B2Z_DP_WARPS; }

cudaError_t launch_zstd_enc_dp(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint32_t* cand, uint8_t* choice,
                               uint64_t* seqs, uint32_t* nseq, uint8_t* lits, uint32_t* nlit, cudaStream_t st) {
    if (srcSize == 0) return cudaSuccess;
    const uint64_t F = 1ull << g.frameLog, nFrames = (srcSize + F - 1) >> g.frameLog;
    const uint32_t nBlockSlots = (uint32_t)(nFrames << (g.frameLog - 17u));
    cudaError_t e = cudaFuncSetAttribute(zstd_enc_dp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)zstd_enc_dp_smem_bytes());
    if (e != cudaSuccess) return e;
    zstd_enc_dp_kernel<<<(nBlockSlots + B2Z_DP_WARPS - 1) / B2Z_DP_WARPS, B2Z_DP_WARPS * 32, zstd_enc_dp_smem_bytes(), st>>>(
        src, srcSize, g, cand, choice, seqs, nseq, lits, nlit, nBlockSlots);
    return cudaGetLastError();
}
#endif

}  // namespace b2z
