// zstd_enc_dp.cu -- stage G of the block-parallel Zstandard encoder (sm_90a): the parse.
//
// One WARP owns one 128 KiB block, one LANE one 4 KiB segment of it (B2Z_SEG): 32 768 blocks x 32 lanes per 4 GiB, so the
// strictly sequential part of the parse -- a minimum-price path -- runs as a million independent chains.  Per block:
//   1. literal prices: byte histogram of the first 64 of every 256 bytes (coalesced 16-byte loads, shared-memory atomics),
//      price = log2(total / count) in 1/16 bit, clamped;
//   2. per lane, a backward dynamic programme over its segment: cost[i] = min(literal + cost[i+1], the position's
//      candidate (stage F) at its length L, L-1, L-2: B2Z_DP_MATCH + offset extra bits + cost[i+l]).  Only the
//      next B2Z_CAP costs are live (candidates are at most B2Z_CAP long), kept in a per-lane ring in shared memory, cost[i+1]
//      also in a register, and the match price is formed four positions ahead of the chain (dp_match); the choice (0 = literal,
//      else the length) goes to a byte array in HBM, four positions per store;
//   3. per lane, one forward walk over the path: a chosen match of the full B2Z_CAP bytes is extended by direct comparison
//      to the segment end, each match becomes its (offBase, litLength, matchLength) record, staged at the lane's own run of
//      the block's sequence array, and each tile's path literals become a 32-bit mask, kept where the tile's choices were.
//      The repcode history is "unknown" at every segment start, so no lane waits for another; only the first record's
//      literal length depends on the lanes before;
//   4. warp scans turn the counts into each lane's place in the block's sequence and literal arrays and into the literal
//      run that reaches into a lane from the lanes before it;
//   5. the move packs the staged records behind each other and completes each lane's first literal length;
//   6. the literal bytes, from the source tiles and the masks (a tile's literals one lane's run per store, dp_emit_literals).
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
// The walk stages lane j's records at out + DP_LANE_SEQS * j (a match is at least B2Z_DP_MINLEN long), and the move packs them
// behind each other once the warp scan has placed every lane.
constexpr uint32_t DP_LANE_SEQS = B2Z_SEG / B2Z_DP_MINLEN;
static_assert(32u * DP_LANE_SEQS <= B2Z_MAXSEQ, "every lane's records fit its staging run in the block's sequence array");
// records a lane keeps in shared memory between stores: at most 8 start in one tile (32 positions / B2Z_DP_MINLEN), and the warp stores
// them once a lane holds more than 8
constexpr uint32_t DP_PEND = 16;
static_assert(32u / B2Z_DP_MINLEN <= DP_PEND / 2u, "a tile's records fit behind the ones a lane may still hold");
struct DpWarpSmem {
    union {
        uint32_t ring[DP_RING][32];  // programme: cost ring [position & (DP_RING - 1)][lane]; a candidate reaches at most B2Z_CAP positions ahead
        uint64_t recs[32][DP_PEND];  // walk: [lane][record ^ (lane & 15)] (the swizzle keeps the walk's writes and the stores' reads conflict-free)
        uint32_t runs[3][33];        // move: per lane its first record's place, the distance back from its staging run, its literal-length patch
    };
    uint32_t candTile[32][33];   // [lane][position in tile]; the byte histogram (256 words) lives here before the first tile
    uint32_t srcTile[32][9];     // [lane][4 input bytes]; the walk keeps the path-literal masks of up to 8 tiles here
    uint32_t chcTile[32][9];     // [lane][4 choices]; the literal pass reads the masks back into it
    uint8_t litc[256];
};

// -DB2Z_DP_CLOCKS (off by default; tools/enc_parse_profile.py --build-clocks): every warp adds the clock64() cycles it spends in each
// phase to dp_clocks[]; b200z_dp_clocks() reads and clears them.  Without the switch the ticks compile to nothing.
enum { DPC_HIST, DPC_DP_LOAD, DPC_DP, DPC_DP_STORE, DPC_WALK_LOAD, DPC_WALK, DPC_WALK_STORE, DPC_SCAN, DPC_MOVE, DPC_LIT_LOAD, DPC_LIT, DPC_N };
#ifdef B2Z_DP_CLOCKS
__device__ unsigned long long dp_clocks[DPC_N + 1];                         // [DPC_N] = warps
#define DP_TICK(ph) do { const long long now_ = clock64(); dpc[ph] += (unsigned long long)(now_ - dpLast); dpLast = now_; } while (0)
#define DP_CLOCKS_FLUSH() do { if (lane == 0) { for (int p_ = 0; p_ < DPC_N; p_++) atomicAdd(&dp_clocks[p_], dpc[p_]); atomicAdd(&dp_clocks[DPC_N], 1ull); } } while (0)
#else
#define DP_TICK(ph) do { } while (0)
#define DP_CLOCKS_FLUSH() do { } while (0)
#endif

// 16 * log2(x) as b2z_zstd_cost.h:zop_log16, with the fraction table in registers
__device__ __forceinline__ uint32_t dp_log16(uint32_t x) {
    const uint32_t hb = highbit32(x);
    const uint32_t k = hb >= 4u ? ((x >> (hb - 4u)) & 15u) : ((x << (4u - hb)) & 15u);
    // ZOP_FRAC_LIST (1,2,3,5,6,7,8,9 | 10,11,12,13,14,15,15,16) as two words of bytes
    const uint64_t lo = 0x0908070605030201ull, hi = 0x100F0F0E0D0C0B0Aull;
    const uint32_t fr = (uint32_t)(((k < 8u ? lo : hi) >> ((k & 7u) * 8u)) & 0xFFu);
    return 16u * hb + ((k == 0u && (x & (x - 1u)) == 0u) ? 0u : fr);
}

// Tiles are fetched into registers one tile ahead of the pass that uses them (fetch t+1 -- or t-1 in the backward DP -- right after
// putting tile t into shared memory), so a tile's loads are in flight while the warp works on the one before: r[j] = row j's word in
// column `lane`: 40 registers per lane in the DP pass and the walk, 16 in the literal pass.  A second set of shared-memory tiles
// would cost 5.4 KB per warp.
// tile t of a 32-bit-per-position array: 32 coalesced 128-byte rows, all issued at once.  base = the block's array, bn = positions in the block
__device__ __forceinline__ void dp_fetch_cand(uint32_t (&r)[32], const uint32_t* __restrict__ base, uint32_t bn, uint32_t t, uint32_t lane) {
#pragma unroll
    for (uint32_t j = 0; j < 32u; j++) {
        const uint32_t pos = j * B2Z_SEG + 32u * t + lane;
        r[j] = pos < bn ? __ldcs(base + pos) : 0u;
    }
}
__device__ __forceinline__ void dp_put_cand(DpWarpSmem& sm, const uint32_t (&r)[32], uint32_t lane) {
#pragma unroll
    for (uint32_t j = 0; j < 32u; j++) sm.candTile[j][lane] = r[j];
}
// tile t of a byte-per-position array: 8 loads of 4 rows x 32 bytes.  WRITTEN: the words were stored earlier in this kernel (the
// path-literal masks), so they are read through L2 (__ldcg) and not through the non-coherent cache
template <bool WRITTEN = false>
__device__ __forceinline__ void dp_fetch_bytes(uint32_t (&r)[8], const uint8_t* __restrict__ base, uint32_t bn, uint32_t t, uint32_t lane) {
#pragma unroll
    for (uint32_t k = 0; k < 8u; k++) {
        const uint32_t row = 4u * k + (lane >> 3), wd = lane & 7u, pos = row * B2Z_SEG + 32u * t + 4u * wd;
        const uint32_t* const p = reinterpret_cast<const uint32_t*>(base + pos);
        r[k] = pos < bn ? (WRITTEN ? __ldcg(p) : __ldg(p)) : 0u;
    }
}
__device__ __forceinline__ void dp_put_bytes(uint32_t (*tile)[9], const uint32_t (&r)[8], uint32_t lane) {
#pragma unroll
    for (uint32_t k = 0; k < 8u; k++) tile[4u * k + (lane >> 3)][lane & 7u] = r[k];
}
__device__ __forceinline__ void dp_store_byte_tile(const uint32_t (*tile)[9], uint8_t* __restrict__ base, uint32_t bn, uint32_t t, uint32_t lane) {
#pragma unroll
    for (uint32_t r = 0; r < 8u; r++) {
        const uint32_t row = 4u * r + (lane >> 3), wd = lane & 7u, pos = row * B2Z_SEG + 32u * t + 4u * wd;
        if (pos < bn) *reinterpret_cast<uint32_t*>(base + pos) = tile[row][wd];
    }
}

// The match half of step p of the programme (p = position in the tile): the candidate priced at its length L, L-1 .. L-NTRUNC as
// (price << 2 | k), minimum over the lengths that qualify, so a tie goes to the longer one as in the sequential statement's strict
// '<' tests.  mc = the price (2^30 - 1 when no length qualifies: more than any literal path), mh = the length.  Positions past the
// segment end (p >= lim) get price 0 and length 0, which makes the step's cost 0 -- the end's cost -- and its choice a literal.
static_assert(DP_RING == 32u && B2Z_DP_NTRUNC < 4u && (uint64_t)B2Z_SEG * B2Z_DP_LIT_MAX + 1024u < (1u << 29),
              "ring slot = position in the tile; k fits two bits; a cost fits 29 bits");
__device__ __forceinline__ void dp_match(const DpWarpSmem& sm, uint32_t lane, uint32_t p, uint32_t lim, uint32_t& mc, uint32_t& mh) {
    const uint32_t c = sm.candTile[lane][p];
    const uint32_t len = B2Z_CAND_LEN(c), ob = 16u * highbit32(B2Z_CAND_OFF(c) + 3u) + B2Z_DP_MATCH;
    uint32_t m = 0xFFFFFFFFu;
#pragma unroll
    for (uint32_t k = 0; k <= B2Z_DP_NTRUNC; k++) {
        // wraps below zero when len < k: the index stays inside the ring, the price is discarded
        const uint32_t key = ((ob + sm.ring[(p + len - k) & (DP_RING - 1u)][lane]) << 2) | k;
        m = (len >= B2Z_DP_MINLEN + k && key < m) ? key : m;
    }
    mc = p >= lim ? 0u : m >> 2;
    mh = p >= lim ? 0u : len - (m & 3u);
}

// per-lane state of the forward walk over a segment's choices (positions segment-relative)
struct DpWalk {
    uint32_t i, ns, nl, np;                 // position; sequences / literals so far; records not yet stored
    uint32_t prevEnd, rep0, rep1, rep2;     // end of the last match (0 before the first); repcode history
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
// the tile's "choice != 0" mask), and the loop runs once per match instead of once per position.  Each match becomes its final
// (offBase, litLength, matchLength) record in sm.recs, except that the segment's first record counts its literals from the segment
// start: the repcode history is "unknown" (0) there, so that record is coded with its explicit offset whatever the lanes before
// left, and only its literal length waits for the warp scan.  Returns the tile's positions that are literals of the path (bit w =
// position 32 t + w), which dp_emit_literals writes out after the scan.
__device__ __forceinline__ uint32_t dp_walk_tile(DpWarpSmem& sm, DpWalk& k, uint32_t t, uint32_t lane, uint32_t sn,
                                                 const uint64_t* __restrict__ fw /* frame as words */, uint32_t segAbs /* frame-relative */, uint32_t nWords) {
    const uint32_t tEnd = (32u * t + 32u) < sn ? (32u * t + 32u) : sn;
    uint32_t lits = 0;
    if (k.i >= tEnd) return lits;
    const uint32_t inTile = tEnd - 32u * t;
    const uint32_t M = dp_nonzero_mask(sm.chcTile[lane]) & (inTile >= 32u ? 0xFFFFFFFFu : ((1u << inTile) - 1u));
    while (k.i < tEnd) {
        uint32_t w = k.i & 31u;
        const uint32_t rem = M >> w;
        const uint32_t r = rem ? (uint32_t)(__ffs((int)rem) - 1) : (tEnd - k.i);        // literals up to the next match of the tile (or the tile's end)
        if (r) {
            lits |= (0xFFFFFFFFu >> (32u - r)) << w;
            k.nl += r; k.i += r; w += r;
            if (!rem) break;
        }
        uint32_t l = (sm.chcTile[lane][w >> 2] >> (8u * (w & 3u))) & 255u;
        const uint32_t off = B2Z_CAND_OFF(sm.candTile[lane][w]);
        if (l == B2Z_CAP) l = match_len(fw, segAbs + k.i - off, segAbs + k.i, sn - k.i, nWords);   // the full common prefix, to the segment end at most
        const uint32_t ll = k.i - k.prevEnd;
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
        sm.recs[lane][k.np ^ (lane & 15u)] = B2Z_PACK_SEQ(offBase, ll, l);
        k.np++; k.ns++; k.i += l; k.prevEnd = k.i;
    }
    return lits;
}

// the records the lanes hold in sm.recs, two lanes' runs per warp store (lane L's due at out + DP_LANE_SEQS L + its count before them);
// the walk's writes must be synced
__device__ __forceinline__ void dp_store_records(const DpWarpSmem& sm, DpWalk& k, uint32_t lane, uint64_t* __restrict__ out) {
    static_assert(DP_PEND == 16u, "a half-warp stores one lane's run");
    const uint32_t from = DP_LANE_SEQS * lane + k.ns - k.np, r = lane & 15u;
#pragma unroll 4
    for (uint32_t s = 0; s < 16u; s++) {
        const uint32_t L = 2u * s + (lane >> 4);
        const uint32_t cnt = __shfl_sync(B2Z_FULL, k.np, L), at = __shfl_sync(B2Z_FULL, from, L);
        if (r < cnt) out[at + r] = sm.recs[L][r ^ (L & 15u)];
    }
    k.np = 0;
}

// the literals of one tile, lane by lane: lane L's are the bytes of its source row where bit `lits` is set, due at out + dst (its
// place in the block's literal array); lane j of the warp writes byte j when it is one, so each store covers one lane's run in
// one or two sectors instead of 32 lanes' bytes in 32 lines.  The source rows must be in shared memory (synced).
__device__ __forceinline__ void dp_emit_literals(const DpWarpSmem& sm, uint32_t lits, uint32_t dst, uint32_t lane, uint8_t* __restrict__ out) {
    const uint32_t below = (1u << lane) - 1u;
    for (uint32_t L = 0; L < 32u; L++) {
        const uint32_t m = __shfl_sync(B2Z_FULL, lits, L), d = __shfl_sync(B2Z_FULL, dst, L);
        if (m >> lane & 1u) out[d + __popc(m & below)] = (uint8_t)(sm.srcTile[L][lane >> 2] >> (8u * (lane & 3u)));
    }
}

// 4 CTAs (16 warps) per SM: with that budget ptxas keeps 124 registers, and the kernel runs faster than the 96-register, 20-warp
// schedule it picks without the minimum
__global__ void __launch_bounds__(B2Z_DP_WARPS * 32, 4)
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
#ifdef B2Z_DP_CLOCKS
    unsigned long long dpc[DPC_N] = {};
    long long dpLast = clock64();
#endif

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
    DP_TICK(DPC_HIST);

    // ---- 2. backward dynamic programme, tile by tile from the segment's end
    const uint32_t s0 = lane * B2Z_SEG;
    const bool active = s0 < bn;
    const uint32_t sn = active ? ((bn - s0) < B2Z_SEG ? (bn - s0) : B2Z_SEG) : 0u;
    uint32_t diff = 0;                                                         // any byte of the segment unlike the block's first byte
    const uint32_t first = bs[0];
    const uint32_t first4 = first * 0x01010101u;
    uint32_t c1 = 0;                                                           // cost[i + 1]: 0 at the segment's end
    if (active) sm.ring[sn & (DP_RING - 1u)][lane] = 0;
    uint32_t cr[32], sr[8];                                                    // the next tile's loads
    dp_fetch_cand(cr, cndB, bn, nTiles - 1u, lane);
    dp_fetch_bytes(sr, bs, bn, nTiles - 1u, lane);
    for (uint32_t t = nTiles; t-- > 0;) {
        dp_put_cand(sm, cr, lane);
        dp_put_bytes(sm.srcTile, sr, lane);
        if (t) { dp_fetch_cand(cr, cndB, bn, t - 1u, lane); dp_fetch_bytes(sr, bs, bn, t - 1u, lane); }
        __syncwarp();
        DP_TICK(DPC_DP_LOAD);
        if (32u * t < sn) {
            // Each step is cost[i] = min(literal + cost[i + 1], the match price), with cost[i + 1] in a register.  The match price
            // only reads cost[i + B2Z_DP_MINLEN ..], so it is formed four positions ahead (mc, mh: price and length), right after
            // the cost it needs last was stored, and its ring loads are in flight while the chain runs three more steps.
            const uint32_t lim = sn - 32u * t;                                 // positions of the tile in the segment (>= 32: all)
            uint32_t mc[4], mh[4];                                             // [j]: position 4 wi + 3 - j
#pragma unroll
            for (uint32_t j = 0; j < 4u; j++) dp_match(sm, lane, 31u - j, lim, mc[j], mh[j]);
#pragma unroll 2
            for (int wi = 7; wi >= 0; wi--) {
                const uint32_t b4 = sm.srcTile[lane][wi];
                const int inWord = (int)lim - 4 * wi;                          // bytes of the word inside the segment
                const uint32_t x = b4 ^ first4;
                diff |= inWord >= 4 ? x : (inWord > 0 ? x & ((1u << (8 * inWord)) - 1u) : 0u);
                uint32_t packed = 0;
#pragma unroll
                for (uint32_t j = 0; j < 4u; j++) {
                    const uint32_t p = 4u * (uint32_t)wi + 3u - j, sh = 8u * (3u - j);
                    const uint32_t lc = c1 + sm.litc[(b4 >> sh) & 255u];
                    c1 = lc < mc[j] ? lc : mc[j];                              // the literal wins a tie
                    packed |= (mc[j] < lc ? mh[j] : 0u) << sh;
                    sm.ring[p][lane] = c1;                                     // p = i & (DP_RING - 1)
                    if (wi > 0) dp_match(sm, lane, p - 4u, lim, mc[j], mh[j]);
                }
                sm.chcTile[lane][wi] = packed;
            }
        }
        __syncwarp();
        DP_TICK(DPC_DP);
        dp_store_byte_tile(sm.chcTile, chcB, bn, t, lane);
        DP_TICK(DPC_DP_STORE);
    }
    // ---- one repeated byte: the canonical single sequence (stage E emits an RLE block for it)
    if (!__any_sync(B2Z_FULL, diff != 0u) && bn > 1u) {
        if (lane == 0) { out[0] = B2Z_PACK_SEQ(1u + 3u, 1u, bn - 1u); lit[0] = bs[0]; nseq[bw] = 1u; nlit[bw] = 1u; }
        DP_CLOCKS_FLUSH();
        return;
    }

    const uint64_t* __restrict__ fw = reinterpret_cast<const uint64_t*>(fb);
    const uint32_t nWords = (n + 7u) >> 3;
    // ---- 3. the walk (tile 0's choices and candidates are still in shared memory from the last step of the programme)
    DpWalk k; k.i = 0; k.ns = 0; k.nl = 0; k.np = 0; k.prevEnd = 0; k.rep0 = k.rep1 = k.rep2 = 0;
    uint32_t qr[8];
    for (uint32_t t = 0; t < nTiles; t++) {
        if (t) { dp_put_bytes(sm.chcTile, qr, lane); dp_put_cand(sm, cr, lane); __syncwarp(); }
        if (t + 1u < nTiles) { dp_fetch_bytes(qr, chcB, bn, t + 1u, lane); dp_fetch_cand(cr, cndB, bn, t + 1u, lane); }
        DP_TICK(DPC_WALK_LOAD);
        sm.srcTile[lane][t & 7u] = dp_walk_tile(sm, k, t, lane, sn, fw, b0 + s0, nWords);
        __syncwarp();
        DP_TICK(DPC_WALK);
        // the masks of tiles 8 u .. 8 u + 7 go where tile 8 u's choices were (each lane's 32 bytes: every tile's mask has a place there)
        if ((t & 7u) == 7u || t + 1u == nTiles) dp_store_byte_tile(sm.srcTile, chcB, bn, t & ~7u, lane);
        if (__any_sync(B2Z_FULL, k.np > DP_PEND / 2u) || t + 1u == nTiles) { dp_store_records(sm, k, lane, out); __syncwarp(); }
        DP_TICK(DPC_WALK_STORE);
    }
    const uint32_t cntSeq = k.ns, cntLit = k.nl;
    // ---- 4. places: exclusive sums of the counts, exclusive maximum of the last match ends
    uint32_t seqBase = cntSeq, litBase = cntLit, prevEnd = cntSeq ? s0 + k.prevEnd : 0u;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t a = __shfl_up_sync(B2Z_FULL, seqBase, d), c = __shfl_up_sync(B2Z_FULL, litBase, d), e = __shfl_up_sync(B2Z_FULL, prevEnd, d);
        if (lane >= (uint32_t)d) { seqBase += a; litBase += c; prevEnd = e > prevEnd ? e : prevEnd; }
    }
    const uint32_t totSeq = __shfl_sync(B2Z_FULL, seqBase, 31), totLit = __shfl_sync(B2Z_FULL, litBase, 31);
    seqBase -= cntSeq; litBase -= cntLit;
    prevEnd = __shfl_up_sync(B2Z_FULL, prevEnd, 1); if (lane == 0) prevEnd = 0;
    sm.runs[0][lane] = seqBase; sm.runs[1][lane] = DP_LANE_SEQS * lane - seqBase; sm.runs[2][lane] = s0 - prevEnd;
    if (lane == 0) sm.runs[0][32] = totSeq;
    __syncwarp();
    DP_TICK(DPC_SCAN);
    // ---- 5. the move: record r of the block comes from its lane's staging run, r + runs[1][lane] (never below r, so a round's loads
    // precede any store over them), and the lane's first record gets the literals before the segment start
    {
        constexpr uint32_t U = 8;
        uint32_t L = 0;                                                        // the last lane whose run starts at or before r
        for (uint32_t c = 0; c < totSeq; c += 32u * U) {
            uint64_t v[U];
            uint32_t patch[U];                                                 // added after the loads, which stay in flight together
#pragma unroll
            for (uint32_t u = 0; u < U; u++) {
                const uint32_t r = c + 32u * u + lane;
                patch[u] = 0;
                if (r < totSeq) {
                    while (sm.runs[0][L + 1u] <= r) L++;                       // runs[0][32] = totSeq ends the search
                    v[u] = __ldcg(out + r + sm.runs[1][L]);
                    if (r == sm.runs[0][L]) patch[u] = sm.runs[2][L];          // s0 - prevEnd more literals
                }
            }
            __syncwarp();
#pragma unroll
            for (uint32_t u = 0; u < U; u++) {
                const uint32_t r = c + 32u * u + lane;
                if (r < totSeq) out[r] = v[u] + ((uint64_t)patch[u] << 28);   // litLength field
            }
        }
    }
    DP_TICK(DPC_MOVE);
    // ---- 6. the literals: each tile's path literals from its mask, in place after the literals of the tiles before
    uint32_t litAt = litBase;
    dp_fetch_bytes(sr, bs, bn, 0, lane);
    dp_fetch_bytes<true>(qr, chcB, bn, 0, lane);
    for (uint32_t t = 0; t < nTiles; t++) {
        if ((t & 7u) == 0u) {
            dp_put_bytes(sm.chcTile, qr, lane);
            if (t + 8u < nTiles) dp_fetch_bytes<true>(qr, chcB, bn, t + 8u, lane);
        }
        dp_put_bytes(sm.srcTile, sr, lane);
        if (t + 1u < nTiles) dp_fetch_bytes(sr, bs, bn, t + 1u, lane);
        __syncwarp();
        DP_TICK(DPC_LIT_LOAD);
        const uint32_t lits = sm.chcTile[lane][t & 7u];
        dp_emit_literals(sm, lits, litAt, lane, lit);
        litAt += __popc(lits);
        __syncwarp();
        DP_TICK(DPC_LIT);
    }
    if (lane == 0) { nseq[bw] = totSeq; nlit[bw] = totLit; }
    DP_CLOCKS_FLUSH();
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

#if defined(B2Z_DP_CLOCKS) && !defined(B2Z_CUEMU)
// the per-phase cycle sums of every warp since the last call (DPC_* order, then the warp count); clears them
extern "C" int b200z_dp_clocks(unsigned long long* out) {
    static const unsigned long long zero[DPC_N + 1] = {};
    cudaError_t e = cudaMemcpyFromSymbol(out, dp_clocks, sizeof(dp_clocks));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(dp_clocks, zero, sizeof(dp_clocks));
    return (int)e;
}
#endif

}  // namespace b2z
