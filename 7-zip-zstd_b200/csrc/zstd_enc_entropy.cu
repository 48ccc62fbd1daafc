// zstd_enc_entropy.cu -- stage E of the block-parallel Zstandard encoder (sm_90a).
//
// Stage E turns stage G's (or stage Z's) output for every 128 KiB block -- final sequences + literal bytes -- into a complete
// zstd block (3-byte header + literals section + sequences section) in the block's slot.  It runs as three kernels:
//   E1 (zstd_enc_tables_kernel, one warp per block): RLE-block test, literal histogram, Huffman code and description, the
//      whole literals section (with the raw and RLE fallbacks), the code histograms, the three mode/table choices, NCount
//      headers, the sequence-section header and the size bound.  The table work is warp-wide: present symbols ranked by
//      compares, one symbol per lane for normalisation and costs, the FSE spread numbered by ballots, the state fill
//      ranked by __match_any_sync.  Blocks that need no FSE chain (RLE blocks, no sequences, over the bound) are finished
//      here; every other block leaves an EntRec (header sizes, logs, the three encoding tables) in scratch.
//      Its sequence pass also leaves the three codes of every sequence (LL | OF << 8 | ML << 16) in the block's word area.
//   E2 (zstd_enc_chains_kernel, one block per lane, ENT_CHAIN_BLOCKS per one-warp CTA): a lane runs the LL, OF and ML state
//      chains of its block together from the last sequence to the first, reading the code words, and writes over each one
//      word per sequence: the three states' bits in stream order (OF, ML, LL; <= 26 bits) and their count.
//   E3 (zstd_enc_seqbits_kernel, one warp per block): the sequence bitstream -- state word + LL/ML/OF extra bits per
//      sequence, placed by prefix sum -- then the final states, the end mark, and the compressed-or-raw block choice.
//
// Replaces (reference, /root/reference/C/zstd/): zstd_compress.c:2888
// (ZSTD_entropyCompressSeqStore_internal), zstd_compress_literals.c:129-235, hist.c:164,
// huf_compress.c:755,248,1167, zstd_compress.c:2693,2763, zstd_compress_sequences.c:156,242,291,
// fse_compress.c:68,330,465.  The sequential statement of exactly this algorithm is
// oracle/zstd_enc_oracle.c (write_literals / write_sequences / compress_block); every
// decision is integer and mirrors it, so the bytes must be identical.
#include "b2z_device.cuh"
#include "b2z_kernels.h"

namespace b2z {

// ---------------------------------------------------------------- format constants
__device__ const uint32_t d_LL_base[36] = { 0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,
    16,18,20,22,24,28,32,40,48,64,0x80,0x100,0x200,0x400,0x800,0x1000,0x2000,0x4000,0x8000,0x10000 };
__device__ const uint8_t d_LL_bits[36] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
    1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16 };
__device__ const uint32_t d_ML_base[53] = { 3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,
    19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,
    35,37,39,41,43,47,51,59,67,83,99,0x83,0x103,0x203,0x403,0x803,0x1003,0x2003,0x4003,0x8003,0x10003 };
__device__ const uint8_t d_ML_bits[53] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
    0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
    1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16 };
__device__ const int16_t d_LL_defNorm[36] = { 4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,
    2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1 };
__device__ const int16_t d_ML_defNorm[53] = { 1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,
    1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,
    1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1 };
__device__ const int16_t d_OF_defNorm[29] = { 1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,
    1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1 };
__device__ const uint8_t d_log2frac[32] = { 0, 11, 22, 33, 43, 53, 63, 72, 82, 91, 100, 108, 116, 125, 132, 140,
    148, 155, 162, 169, 176, 182, 189, 195, 201, 207, 213, 219, 225, 230, 236, 241 };

// length codes (RFC 8878 3.1.1.3.2.1.1): a table below 64 (literal lengths) and 128 (match lengths - 3), the highest set bit above
__device__ const uint8_t d_LL_code[64] = { 0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,16,17,17,18,18,19,19,20,20,20,20,21,21,21,21,
    22,22,22,22,22,22,22,22,23,23,23,23,23,23,23,23,24,24,24,24,24,24,24,24,24,24,24,24,24,24,24,24 };
__device__ const uint8_t d_ML_code[128] = { 0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,19,20,21,22,23,24,25,26,27,28,29,30,31,
    32,32,33,33,34,34,35,35,36,36,36,36,37,37,37,37,38,38,38,38,38,38,38,38,39,39,39,39,39,39,39,39,
    40,40,40,40,40,40,40,40,40,40,40,40,40,40,40,40,41,41,41,41,41,41,41,41,41,41,41,41,41,41,41,41,
    42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42,42 };
__device__ __forceinline__ uint32_t ll_code(uint32_t ll) { return ll < 64 ? (uint32_t)d_LL_code[ll] : highbit32(ll) + 19u; }
__device__ __forceinline__ uint32_t ml_code(uint32_t m) { return m < 128 ? (uint32_t)d_ML_code[m] : highbit32(m) + 36u; }   // m = matchLength - 3

// -DB2Z_E_CLOCKS (off by default; tools/enc_entropy_profile.py --build-clocks): lane 0 of every E1 and E2 warp adds the clock64()
// cycles its warp spends in each phase to e_clocks[]; b200z_e_clocks() reads and clears them.  E1: literal histogram (with the
// RLE-block test), Huffman build and description, literal streams (or the raw / RLE literals), sequence pass (code histograms),
// the three table choices, table hand-off (or the block's finish).  E2: table staging, code loads, chain steps, word stores.
// Without the switch the ticks compile to nothing.
enum { E1C_LITHIST, E1C_HUF, E1C_LITSTREAMS, E1C_SEQPASS, E1C_TABLES, E1C_HANDOFF, E1C_N };
enum { E2C_STAGE, E2C_LOAD, E2C_STEP, E2C_STORE, E2C_N };
#if defined(B2Z_E_CLOCKS) && !defined(B2Z_CUEMU)
__device__ unsigned long long e_clocks[E1C_N + E2C_N];                  // E1's phases, then E2's
#define E_CLOCKS_START(n) unsigned long long ec_[n] = {}; long long ecLast_ = clock64()
#define E_TICK(ph) do { const long long now_ = clock64(); ec_[ph] += (unsigned long long)(now_ - ecLast_); ecLast_ = now_; } while (0)
#define E_CLOCKS_FLUSH(base, n) do { if (lane == 0) for (int p_ = 0; p_ < (n); p_++) atomicAdd(&e_clocks[(base) + p_], ec_[p_]); } while (0)
#else
#define E_CLOCKS_START(n) do { } while (0)
#define E_TICK(ph) do { } while (0)
#define E_CLOCKS_FLUSH(base, n) do { } while (0)
#endif

__device__ __forceinline__ uint32_t warp_sum(uint32_t v) {
    for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(B2Z_FULL, v, d);
    return v;
}
__device__ __forceinline__ uint32_t warp_max(uint32_t v) {
    for (int d = 16; d; d >>= 1) { const uint32_t o = __shfl_xor_sync(B2Z_FULL, v, d); v = o > v ? o : v; }
    return v;
}

// ---------------------------------------------------------------- per-warp workspace of E1
struct FseCT {                       // FSE encoding table of one symbol type
    uint16_t state[512];
    int32_t  dfs[64];                // deltaFindState
    uint32_t dnb[64];                // deltaNbBits
    uint32_t log;
};

#define STAGE_WORDS 384
#define STAGE_FLUSH_BITS (STAGE_WORDS * 32 - 3072)

struct WarpWS {
    uint32_t hist[256];              // literal byte counts; later LL/OF/ML code counts at [0],[64],[128]
    uint16_t hufCode[256];
    uint8_t  hufLen[256];
    union {
        struct { uint32_t w[512]; uint16_t parent[512]; uint8_t order[256]; uint8_t depth[512]; uint32_t key[256]; } hb;   // Huffman build
        struct { FseCT ct[3]; } fse;                                                                                        // LL, OF, ML
    } u;
    uint8_t  spread[512];            // FSE symbol spreading scratch
    int16_t  norm[64];
    uint16_t cumul[66];              // FSE build: first state slot of each symbol, then its running fill position
    uint16_t cpos[66];               // FSE build: first spread index of each symbol with a positive count
    uint32_t rk[16], rstart[16], rnext[16];   // Huffman canonical codes: symbols per rank, first code, codes given so far
    uint32_t wcnt[16];               // Huffman weight counts
    uint32_t stage[STAGE_WORDS];     // bit staging window
};

// ---------------------------------------------------------------- E1 -> E2 -> E3 record, one per block in scratch
// The three encoding tables in the layout E2 keeps in shared memory: states LL | OF | ML, then {deltaNbBits, deltaFindState}
// per symbol LL | OF | ML.
#define ENT_ST_OF 512u
#define ENT_ST_ML 768u
#define ENT_ST_N  1280u
#define ENT_SY_OF 36u
#define ENT_SY_ML 68u
#define ENT_SY_N  121u
struct EntTables {
    uint16_t state[ENT_ST_N];
    uint2    sym[ENT_SY_N];
    uint32_t pad[2];
};
struct EntRec {
    uint32_t run;                    // 1: E2 and E3 code this block's sequences; 0: E1 finished the block
    uint32_t bodyHead;               // bytes of the block body before the sequence bitstream
    uint32_t logs;                   // table logs: LL | OF << 8 | ML << 16
    uint32_t pad0;
    uint16_t fin[4];                 // final states LL, OF, ML (written by E2)
    uint32_t pad1[2];
    EntTables tab;
};
static_assert(sizeof(EntTables) % 16 == 0 && sizeof(EntRec) % 16 == 0 && offsetof(EntRec, tab) % 16 == 0, "EntRec is copied in 16-byte units");
#define ENT_SCRATCH_STRIDE ((size_t)sizeof(EntRec) + (size_t)B2Z_MAXSEQ * 4u)   // record, then one word per sequence (E1: codes, E2: states)
static_assert(sizeof(EntRec) + (size_t)B2Z_MAXSEQ * 4u <= (size_t)B2Z_BLOCK * 4u, "stage E scratch must fit the block's candidate words");

// ---------------------------------------------------------------- lane-0 bit writer to global memory
struct BitW {
    uint8_t* p; uint64_t acc; uint32_t nb;
    __device__ __forceinline__ void init(uint8_t* q) { p = q; acc = 0; nb = 0; }
    __device__ __forceinline__ void add(uint32_t v, uint32_t n) {
        acc |= (uint64_t)(v & (n >= 32 ? 0xFFFFFFFFu : ((1u << n) - 1u))) << nb; nb += n;
        while (nb >= 8) { *p++ = (uint8_t)acc; acc >>= 8; nb -= 8; }
    }
    __device__ __forceinline__ uint8_t* close() { add(1, 1); if (nb) { *p++ = (uint8_t)acc; acc = 0; nb = 0; } return p; }
    __device__ __forceinline__ uint8_t* flush_partial() { if (nb) { *p++ = (uint8_t)acc; acc = 0; nb = 0; } return p; }
};

// ---------------------------------------------------------------- FSE (warp-wide unless noted)
// Encoding table of `norm` (symbols 0..maxSym, maxSym < 64, log >= 5).  The serial statement spreads the symbols in order
// over positions k*step & mask (k = 0, 1, ...), skipping those above `high` where the "less than 1" symbols sit; step is odd,
// so every position is visited once, and the m-th accepted position takes the m-th slot of the symbols' count runs.
__device__ void fse_build_ctable(WarpWS* ws, FseCT* ct, const int16_t* norm, uint32_t maxSym, uint32_t log, uint32_t lane) {
    const uint32_t size = 1u << log, mask = size - 1u, step = (size >> 1) + (size >> 3) + 3u, lt = (1u << lane) - 1u;
    uint16_t* cumul = ws->cumul; uint16_t* cpos = ws->cpos; uint8_t* spread = ws->spread;
    uint32_t cu = 0, cp = 0, nLow = 0;
    for (uint32_t s0 = 0; s0 <= maxSym; s0 += 32) {
        const uint32_t s = s0 + lane;
        const int n = s <= maxSym ? norm[s] : 0;
        uint32_t tc, tp;
        const uint32_t ec = warp_excl_scan(n == -1 ? 1u : (n > 0 ? (uint32_t)n : 0u), lane, &tc);
        const uint32_t ep = warp_excl_scan(n > 0 ? (uint32_t)n : 0u, lane, &tp);
        const uint32_t low = __ballot_sync(B2Z_FULL, n == -1);
        if (s <= maxSym) {
            const uint32_t total = cu + ec;
            cumul[s] = (uint16_t)total; cpos[s] = (uint16_t)(cp + ep);
            if (n == 0) { ct->dnb[s] = ((log + 1u) << 16) - size; ct->dfs[s] = 0; }
            else if (n == 1 || n == -1) { ct->dnb[s] = (log << 16) - size; ct->dfs[s] = (int32_t)total - 1; }
            else {
                const uint32_t maxBitsOut = log - highbit32((uint32_t)n - 1u), minStatePlus = (uint32_t)n << maxBitsOut;
                ct->dnb[s] = (maxBitsOut << 16) - minStatePlus;
                ct->dfs[s] = (int32_t)total - n;
            }
            if (n == -1) spread[size - 1u - nLow - (uint32_t)__popc(low & lt)] = (uint8_t)s;
        }
        cu += tc; cp += tp; nLow += (uint32_t)__popc(low);
    }
    __syncwarp();
    const uint32_t high = size - 1u - nLow;
    uint32_t m0 = 0;
    for (uint32_t k0 = 0; k0 < size; k0 += 32) {
        const uint32_t k = k0 + lane, pos = (k * step) & mask;
        const bool acc = k < size && pos <= high;
        const uint32_t bal = __ballot_sync(B2Z_FULL, acc);
        if (acc) {
            const uint32_t m = m0 + (uint32_t)__popc(bal & lt);
            uint32_t lo = 0, hi = maxSym + 1u;                   // the last symbol whose run starts at or before m
            while (hi - lo > 1u) { const uint32_t mid = (lo + hi) >> 1; if (cpos[mid] <= m) lo = mid; else hi = mid; }
            spread[pos] = (uint8_t)lo;
        }
        m0 += (uint32_t)__popc(bal);
    }
    __syncwarp();
    for (uint32_t u0 = 0; u0 < size; u0 += 32) {                 // state fill in spread order, per symbol
        const uint32_t u = u0 + lane;
        const uint32_t s = u < size ? spread[u] : 0xFFFFu;
        const uint32_t grp = __match_any_sync(B2Z_FULL, s);
        if (u < size) ct->state[cumul[s] + (uint32_t)__popc(grp & lt)] = (uint16_t)(size + u);
        __syncwarp();
        if (u < size && (grp >> lane) == 1u) cumul[s] = (uint16_t)(cumul[s] + __popc(grp));
        __syncwarp();
    }
    if (lane == 0) ct->log = log;
    __syncwarp();
}
__device__ __forceinline__ uint32_t fse_init_state(const FseCT* ct, uint32_t sym) {
    const uint32_t nb = (ct->dnb[sym] + (1u << 15)) >> 16;
    const uint32_t v = (nb << 16) - ct->dnb[sym];
    return ct->state[(v >> nb) + ct->dfs[sym]];
}
__device__ __forceinline__ uint32_t fse_encode(const FseCT* ct, uint32_t* state, uint32_t sym, uint32_t* nbOut) {
    const uint32_t nb = (*state + ct->dnb[sym]) >> 16, bits = *state & ((1u << nb) - 1u);
    *state = ct->state[(*state >> nb) + ct->dfs[sym]];
    *nbOut = nb; return bits;
}

// rounding one symbol per lane, then the settle loop on the (first) largest entry
__device__ void fse_normalize(int16_t* norm, uint32_t log, const uint32_t* count, uint32_t total, uint32_t maxSym, uint32_t lane) {
    const uint32_t size = 1u << log; uint32_t sum = 0;
    for (uint32_t s = lane; s <= maxSym; s += 32) {
        int16_t v = 0;
        if (count[s]) {
            uint64_t p = ((uint64_t)count[s] * size * 2u + total) / (2ull * total);
            if (p < 1) p = 1;
            v = (int16_t)p; sum += (uint32_t)p;
        }
        norm[s] = v;
    }
    int32_t delta = (int32_t)size - (int32_t)warp_sum(sum);
    __syncwarp();
    while (delta != 0) {
        uint32_t key = 0;                                        // (entry, lowest index first)
        for (uint32_t s = lane; s <= maxSym; s += 32) { const uint32_t k = ((uint32_t)norm[s] << 8) | (255u - s); key = k > key ? k : key; }
        key = warp_max(key);
        const uint32_t big = 255u - (key & 255u); const int32_t nbig = (int32_t)(key >> 8);
        int32_t nv;
        if (delta > 0) { nv = nbig + delta; delta = 0; }
        else {
            int32_t take = nbig - 1 < -delta ? nbig - 1 : -delta;
            if (take > (nbig >> 1) && nbig > 2) take = nbig >> 1;
            nv = nbig - take; delta += take;
        }
        __syncwarp();
        if (lane == 0) norm[big] = (int16_t)nv;
        __syncwarp();
    }
}

// lane 0
__device__ uint32_t fse_write_ncount(uint8_t* dst, const int16_t* norm, uint32_t maxSym, uint32_t log) {
    BitW b; b.init(dst);
    b.add(log - 5u, 4);
    int32_t remaining = (int32_t)(1u << log);
    uint32_t s = 0;
    while (remaining > 0 && s <= maxSym) {
        const uint32_t nb = highbit32((uint32_t)remaining + 1u) + 1u;
        const uint32_t T = 1u << (nb - 1u), mx = 2u * T - 1u - ((uint32_t)remaining + 1u);
        const int32_t proba = norm[s++];
        const uint32_t count = (uint32_t)(proba + 1);
        remaining -= proba < 0 ? 1 : proba;
        if (count < mx) b.add(count, nb - 1u);
        else if (count < T) b.add(count, nb);
        else b.add(count + mx, nb);
        if (proba == 0) {
            for (;;) {
                uint32_t run = 0;
                while (run < 3 && s <= maxSym && norm[s] == 0) { run++; s++; }
                b.add(run, 2);
                if (run < 3) break;
            }
        }
    }
    return (uint32_t)(b.flush_partial() - dst);
}

__device__ __forceinline__ uint32_t log2_fx8(uint32_t x) {
    const uint32_t hb = highbit32(x);
    const uint32_t m = hb >= 5 ? (x >> (hb - 5)) & 31u : (x << (5 - hb)) & 31u;
    return (hb << 8) + d_log2frac[m];
}
__device__ uint64_t fse_cost_fx8(const uint32_t* count, const int16_t* norm, uint32_t maxSym, uint32_t log, uint32_t lane) {
    uint64_t c = 0; bool bad = false;
    for (uint32_t s = lane; s <= maxSym; s += 32) {
        if (!count[s]) continue;
        if (norm[s] == 0) { bad = true; continue; }
        const uint32_t n = norm[s] < 0 ? 1u : (uint32_t)norm[s];
        c += (uint64_t)count[s] * ((log << 8) - log2_fx8(n));
    }
    if (__any_sync(B2Z_FULL, bad)) return ~0ull;
    for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(B2Z_FULL, c, d);
    return c;
}

// ---------------------------------------------------------------- Huffman (warp-wide; the tree itself on lane 0)
// code lengths (<= 11) into ws->hufLen / hufCode; returns maxBits, sets *maxSymOut
__device__ uint32_t huf_build(WarpWS* ws, uint32_t lane, uint32_t* maxSymOut) {
    const uint32_t* count = ws->hist;
    uint32_t* w = ws->u.hb.w; uint16_t* parent = ws->u.hb.parent; uint8_t* order = ws->u.hb.order; uint8_t* depth = ws->u.hb.depth;
    uint32_t* key = ws->u.hb.key;
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t n, maxd;
    for (uint32_t k = 0;; k++) {
        // present symbols keyed by (count after k halvings, rounded up; symbol); the rank of a key among them is its place
        // in the stable sort by count
        n = 0;
        for (uint32_t s0 = 0; s0 < 256; s0 += 32) {
            const uint32_t s = s0 + lane, c = count[s];
            const uint32_t bal = __ballot_sync(B2Z_FULL, c != 0);
            if (c) key[n + (uint32_t)__popc(bal & lt)] = (((c + (1u << k) - 1u) >> k) << 8) | s;
            n += (uint32_t)__popc(bal);
        }
        __syncwarp();
        for (uint32_t i = lane; i < n; i += 32) {
            const uint32_t ki = key[i]; uint32_t r = 0;
            for (uint32_t j = 0; j < n; j++) r += key[j] < ki ? 1u : 0u;
            order[r] = (uint8_t)ki; w[r] = ki >> 8;
        }
        __syncwarp();
        uint32_t md = 0;
        if (lane == 0) {                                         // two-queue tree on the sorted weights
            uint32_t li = 0, ii = n, ie = n;
            while ((n - li) + (ie - ii) > 1) {
                uint32_t a, b;
                if (li < n && (ii >= ie || w[li] <= w[ii])) a = li++; else a = ii++;
                if (li < n && (ii >= ie || w[li] <= w[ii])) b = li++; else b = ii++;
                w[ie] = w[a] + w[b]; parent[a] = (uint16_t)ie; parent[b] = (uint16_t)ie; ie++;
            }
            depth[ie - 1] = 0;
            for (int i = (int)ie - 2; i >= 0; i--) depth[i] = (uint8_t)(depth[parent[i]] + 1);
            for (uint32_t i = 0; i < n; i++) if (depth[i] > md) md = depth[i];
        }
        maxd = __shfl_sync(B2Z_FULL, md, 0);
        __syncwarp();
        if (maxd <= 11) break;
    }
    for (uint32_t s = lane; s < 256; s += 32) ws->hufLen[s] = 0;
    if (lane < 16) { ws->rk[lane] = 0; ws->rnext[lane] = 0; }
    __syncwarp();
    for (uint32_t i = lane; i < n; i += 32) ws->hufLen[order[i]] = depth[i];
    __syncwarp();
    uint32_t maxSym = 0;
    for (uint32_t s = lane; s < 256; s += 32) {
        if (count[s]) maxSym = s;
        if (ws->hufLen[s]) atomicAdd(&ws->rk[maxd + 1u - ws->hufLen[s]], 1u);
    }
    maxSym = warp_max(maxSym);
    __syncwarp();
    if (lane == 0) { uint32_t pos = 0; for (uint32_t r = 1; r <= maxd; r++) { ws->rstart[r] = pos; pos += ws->rk[r] << (r - 1u); } }
    __syncwarp();
    // canonical codes: within a rank, in symbol order
    for (uint32_t s0 = 0; s0 < 256; s0 += 32) {
        const uint32_t s = s0 + lane, len = ws->hufLen[s], r = len ? maxd + 1u - len : 0u;
        const uint32_t grp = __match_any_sync(B2Z_FULL, r);
        ws->hufCode[s] = len ? (uint16_t)((ws->rstart[r] >> (r - 1u)) + ws->rnext[r] + (uint32_t)__popc(grp & lt)) : (uint16_t)0;
        __syncwarp();
        if (len && (grp >> lane) == 1u) ws->rnext[r] += (uint32_t)__popc(grp);
        __syncwarp();
    }
    *maxSymOut = maxSym;
    return maxd;
}

// tree description at dst; returns bytes written or 0 (not representable)
__device__ uint32_t huf_write_table(WarpWS* ws, uint8_t* dst, uint32_t maxBits, uint32_t maxSym, uint32_t lane) {
    const uint32_t nw = maxSym;
    uint8_t* wt = ws->u.hb.order;                                // weights (hb scratch is dead now; order[256] reused)
    uint32_t maxW = 0;
    for (uint32_t s = lane; s < nw; s += 32) {
        const uint32_t v = ws->hufLen[s] ? maxBits + 1u - ws->hufLen[s] : 0u;
        wt[s] = (uint8_t)v; maxW = v > maxW ? v : maxW;
    }
    maxW = warp_max(maxW);
    if (lane < 16) ws->wcnt[lane] = 0;
    __syncwarp();
    uint32_t fseSize = 0;
    if (nw > 1) {
        for (uint32_t s = lane; s < nw; s += 32) atomicAdd(&ws->wcnt[wt[s]], 1u);
        __syncwarp();
        const uint32_t maxCnt = warp_max(lane <= maxW ? ws->wcnt[lane] : 0u);
        if (maxCnt != nw && maxCnt > 1) {
            uint32_t log = 6;
            const uint32_t minBits = highbit32(nw) + 1u, symBits = highbit32(maxW + 1u) + 2u;
            const uint32_t lo = minBits < symBits ? minBits : symBits;
            const uint32_t want = highbit32(nw - 1u) >= 2u ? highbit32(nw - 1u) - 2u : 0u;
            if (want < log) log = want;
            if (log < lo) log = lo;
            if (log < 5) log = 5;
            if (log > 6) log = 6;
            int16_t* norm = ws->norm;
            fse_normalize(norm, log, ws->wcnt, nw, maxW, lane);
            uint8_t* tmp = dst + 1;
            uint32_t hs = 0;
            if (lane == 0) hs = fse_write_ncount(tmp, norm, maxW, log);
            hs = __shfl_sync(B2Z_FULL, hs, 0);
            // weights table: a 64-state FseCT carved out of hb.w (dead at this point)
            FseCT* ct = reinterpret_cast<FseCT*>(ws->u.hb.w);
            fse_build_ctable(ws, ct, norm, maxW, log, lane);
            if (lane == 0) {
                BitW b; b.init(tmp + hs);
                uint32_t i = nw, s1, s2, nb, bits;
                if (nw & 1u) { s1 = fse_init_state(ct, wt[--i]); s2 = fse_init_state(ct, wt[--i]);
                               bits = fse_encode(ct, &s1, wt[--i], &nb); b.add(bits, nb); }
                else { s2 = fse_init_state(ct, wt[--i]); s1 = fse_init_state(ct, wt[--i]); }
                while (i > 0) {
                    bits = fse_encode(ct, &s2, wt[--i], &nb); b.add(bits, nb);
                    bits = fse_encode(ct, &s1, wt[--i], &nb); b.add(bits, nb);
                }
                b.add(s2, log); b.add(s1, log);
                fseSize = (uint32_t)(b.close() - tmp);
            }
            fseSize = __shfl_sync(B2Z_FULL, fseSize, 0);
        }
    }
    const uint32_t rawSize = (nw + 1u) / 2u;
    if (fseSize && fseSize < 128u && (fseSize < rawSize || nw > 128u)) { if (lane == 0) dst[0] = (uint8_t)fseSize; return 1u + fseSize; }
    if (nw > 128u || nw == 0u) return 0;
    if (lane == 0) dst[0] = (uint8_t)(127u + nw);
    for (uint32_t i = 2u * lane; i < nw; i += 64) dst[1 + i / 2] = (uint8_t)((wt[i] << 4) | (i + 1 < nw ? wt[i + 1] : 0));
    return 1u + rawSize;
}
static_assert(sizeof(FseCT) <= sizeof(uint32_t) * 512, "weights FseCT must fit in hb.w");

// ---------------------------------------------------------------- warp bit staging
struct Stager {
    uint32_t* stage; uint8_t* out; uint32_t bits;            // uniform: bits currently staged, out = next byte
    __device__ __forceinline__ void init(uint32_t* s, uint8_t* o, uint32_t lane) {
        stage = s; out = o; bits = 0;
        for (uint32_t i = lane; i < STAGE_WORDS; i += 32) stage[i] = 0;
        __syncwarp();
    }
    // OR `nb` (<= 96) bits (lo | hi<<64) at staged bit offset `off`
    __device__ __forceinline__ void put(uint32_t off, uint64_t lo, uint32_t hi, uint32_t nb) {
        if (!nb) return;
        const uint32_t wi = off >> 5, sh = off & 31u;
        const uint32_t w0 = (uint32_t)lo, w1 = (uint32_t)(lo >> 32);
        atomicOr(&stage[wi], w0 << sh);
        const uint32_t end = sh + nb;
        if (end > 32) atomicOr(&stage[wi + 1], sh ? (uint32_t)((((uint64_t)w1 << 32) | w0) >> (32 - sh)) : w1);
        if (end > 64) atomicOr(&stage[wi + 2], sh ? (uint32_t)((((uint64_t)hi << 32) | w1) >> (32 - sh)) : hi);
        if (end > 96) atomicOr(&stage[wi + 3], sh ? (hi >> (32 - sh)) : 0u);
    }
    // write whole bytes out; keep the partial byte (force = also pad the partial byte out)
    __device__ __forceinline__ void flush(uint32_t lane, bool force) {
        __syncwarp();
        const uint32_t nbytes = force ? (bits + 7u) >> 3 : bits >> 3;
        const uint8_t* sb = reinterpret_cast<const uint8_t*>(stage);
        for (uint32_t i = lane; i < nbytes; i += 32) out[i] = sb[i];
        const uint32_t rem = force ? 0u : (bits & 7u);
        const uint32_t carry = rem ? sb[nbytes] : 0u;
        __syncwarp();
        for (uint32_t i = lane; i < STAGE_WORDS; i += 32) stage[i] = (i == 0) ? carry : 0u;
        __syncwarp();
        out += nbytes; bits = rem;
    }
};

// Huffman-encode literals [a, b) as one backward stream at st.out, 4 literals per lane and 128 per step; returns stream bytes
__device__ uint32_t huf_encode_stream(WarpWS* ws, Stager& st, const uint8_t* __restrict__ lit, uint32_t a, uint32_t b, uint32_t lane) {
    uint8_t* start = st.out;
    uint32_t cur[4];                                             // lane's literals hi-1-4*lane .. hi-4-4*lane, loaded a step ahead
#pragma unroll
    for (uint32_t j = 0; j < 4; j++) { const uint32_t k = lane * 4u + j; cur[j] = k < b - a ? lit[b - 1u - k] : 0u; }
    for (uint32_t hi = b; hi > a;) {
        const uint32_t cnt = (hi - a) < 128u ? (hi - a) : 128u, hn = hi - cnt;
        uint32_t nxt[4];
#pragma unroll
        for (uint32_t j = 0; j < 4; j++) { const uint32_t k = lane * 4u + j; nxt[j] = k < hn - a ? lit[hn - 1u - k] : 0u; }
        uint64_t code = 0; uint32_t nb = 0;                      // <= 44 bits
#pragma unroll
        for (uint32_t j = 0; j < 4; j++) {
            const uint32_t k = lane * 4u + j;
            if (k < cnt) { const uint32_t s = cur[j]; code |= (uint64_t)ws->hufCode[s] << nb; nb += ws->hufLen[s]; }
        }
#pragma unroll
        for (uint32_t j = 0; j < 4; j++) cur[j] = nxt[j];
        uint32_t total; const uint32_t off = warp_excl_scan(nb, lane, &total);
        st.put(st.bits + off, code, 0, nb);
        st.bits += total; hi -= cnt;
        if (st.bits > STAGE_FLUSH_BITS) st.flush(lane, false);
    }
    if (lane == 0) st.put(st.bits, 1, 0, 1);                     // end mark
    st.bits += 1;
    st.flush(lane, true);
    return (uint32_t)(st.out - start);
}

__device__ __forceinline__ void warp_copy(uint8_t* dst, const uint8_t* __restrict__ src, uint32_t n, uint32_t lane) {
    for (uint32_t i = lane; i < n; i += 32) dst[i] = src[i];
}

// ---------------------------------------------------------------- sequence table choice (warp-wide)
// returns header bytes written at dst; *mode = 0 predefined, 1 RLE, 2 compressed
__device__ uint32_t choose_seq_table(WarpWS* ws, FseCT* ct, uint8_t* dst, const uint32_t* count, uint32_t nbSeq, uint32_t maxSymAll,
                                     uint32_t maxLog, const int16_t* defNorm, uint32_t defMaxSym, uint32_t defLog, uint32_t* mode, uint32_t lane) {
    uint32_t maxSym = 0, present = 0, big = 0;
    for (uint32_t s = lane; s <= maxSymAll; s += 32) if (count[s]) { maxSym = s; present++; if (count[s] > big) big = count[s]; }
    maxSym = warp_max(maxSym); present = warp_sum(present); big = warp_max(big);
    if (big == nbSeq && !(nbSeq <= 2 && maxSym <= defMaxSym)) {
        for (uint32_t s = lane; s < 64; s += 32) { ct->dnb[s] = 0; ct->dfs[s] = 0; }
        if (lane < 2) ct->state[lane] = 0;
        if (lane == 0) { ct->log = 0; dst[0] = (uint8_t)maxSym; }
        __syncwarp();
        *mode = 1; return 1;
    }
    int16_t* norm = ws->norm;
    // default-table cost (copy default norm into smem for the shared cost routine)
    uint64_t costDef = ~0ull;
    if (maxSym <= defMaxSym) {
        for (uint32_t s = lane; s <= defMaxSym; s += 32) norm[s] = defNorm[s];
        __syncwarp();
        costDef = fse_cost_fx8(count, norm, maxSym, defLog, lane);
        __syncwarp();
    }
    const uint32_t hbN = highbit32(nbSeq > 1 ? nbSeq - 1u : 1u);
    uint32_t log = hbN >= 2 ? hbN - 2u : 0u;
    const uint32_t minA = highbit32(nbSeq) + 1u, minB = highbit32(maxSym ? maxSym : 1u) + 2u, lo = minA < minB ? minA : minB;
    if (log > maxLog) log = maxLog;
    if (log < lo) log = lo;
    if (log < 5) log = 5;
    if (log > maxLog) log = maxLog;
    while ((1u << log) < present) log++;
    fse_normalize(norm, log, count, nbSeq, maxSym, lane);
    uint32_t hs = 0;
    if (lane == 0) hs = fse_write_ncount(dst, norm, maxSym, log);
    hs = __shfl_sync(B2Z_FULL, hs, 0);
    const uint64_t costFse = fse_cost_fx8(count, norm, maxSym, log, lane) + ((uint64_t)hs << 11);
    __syncwarp();
    if (costDef <= costFse || big == nbSeq) {
        for (uint32_t s = lane; s <= defMaxSym; s += 32) norm[s] = defNorm[s];
        __syncwarp();
        fse_build_ctable(ws, ct, norm, defMaxSym, defLog, lane); *mode = 0; return 0;
    }
    fse_build_ctable(ws, ct, norm, maxSym, log, lane); *mode = 2; return hs;
}

// ---------------------------------------------------------------- block geometry
struct BlockGeom { uint32_t blkSize, last; size_t litOff; };   // litOff: the block's offset in the source and literal buffers
__device__ __forceinline__ BlockGeom block_geom(const EncGeom& g, uint64_t srcSize, uint32_t blk) {
    const uint32_t blocksPerFrame = 1u << (g.frameLog - 17u);
    const uint64_t frame = blk / blocksPerFrame; const uint32_t bif = blk % blocksPerFrame;
    const uint64_t f0 = frame << g.frameLog;
    const uint64_t fn = enc_frame_bytes(g, srcSize, frame);
    const uint64_t b0 = (uint64_t)bif << 17;
    BlockGeom r;
    r.blkSize = (uint32_t)((fn - b0) < B2Z_BLOCK ? (fn - b0) : B2Z_BLOCK);
    r.last = (b0 + r.blkSize == fn) ? 1u : 0u;
    r.litOff = (size_t)(f0 + b0);
    return r;
}
__device__ __forceinline__ void put_hdr3(uint8_t* out, uint32_t h) { out[0] = (uint8_t)h; out[1] = (uint8_t)(h >> 8); out[2] = (uint8_t)(h >> 16); }

// the compressed block if it is smaller than the input, else a raw block; returns the slot bytes
__device__ uint32_t finish_block(uint8_t* out, const uint8_t* __restrict__ bsrc, uint32_t blkSize, uint32_t last, uint32_t bodySize, bool overCap, uint32_t lane) {
    if (!overCap && bodySize < blkSize) {
        if (lane == 0) put_hdr3(out, last | (2u << 1) | (bodySize << 3));
        return 3 + bodySize;
    }
    __syncwarp();
    if (lane == 0) put_hdr3(out, last | (blkSize << 3));
    warp_copy(out + 3, bsrc, blkSize, lane);
    return 3 + blkSize;
}

// ---------------------------------------------------------------- E1: tables and literals, one warp per block
__global__ void __launch_bounds__(B2Z_ENT_WARPS * 32)
zstd_enc_tables_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g,
                       const uint64_t* __restrict__ seqs, const uint32_t* __restrict__ nseqArr,
                       const uint8_t* __restrict__ lits, const uint32_t* __restrict__ nlitArr,
                       uint8_t* __restrict__ slots, uint32_t* __restrict__ slotSize, uint8_t* __restrict__ scratch, uint32_t nBlocks) {
    __shared__ WarpWS wsAll[B2Z_ENT_WARPS];
    const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
    WarpWS* ws = &wsAll[wib];
    E_CLOCKS_START(E1C_N);
    for (uint32_t blk = blockIdx.x * B2Z_ENT_WARPS + wib; blk < nBlocks; blk += gridDim.x * B2Z_ENT_WARPS) {
        const BlockGeom bg = block_geom(g, srcSize, blk);
        const uint32_t blkSize = bg.blkSize, last = bg.last;
        const uint8_t* bsrc = src + bg.litOff;
        const uint8_t* lit = lits + bg.litOff;
        const uint64_t* sq = seqs + (size_t)blk * B2Z_MAXSEQ;
        const uint32_t nbSeq = nseqArr[blk], nlit = nlitArr[blk];
        uint8_t* out = slots + (size_t)blk * B2Z_SLOT;
        uint8_t* body = out + 3;
        EntRec* rec = reinterpret_cast<EntRec*>(scratch + (size_t)blk * ENT_SCRATCH_STRIDE);

        // RLE block?
        bool rle = false;
        if (blkSize > 1 && nbSeq == 1 && nlit == 1) {
            const uint64_t s0 = sq[0];
            rle = B2Z_SEQ_LL(s0) == 1 && B2Z_SEQ_ML(s0) == blkSize - 1u && B2Z_SEQ_OFFBASE(s0) == 4u;
        }
        if (rle) {
            if (lane == 0) { put_hdr3(out, last | (1u << 1) | (blkSize << 3)); out[3] = bsrc[0]; slotSize[blk] = 4; rec->run = 0; }
            continue;
        }

        // =========================== literals section
        for (uint32_t i = lane; i < 256; i += 32) ws->hist[i] = 0;
        __syncwarp();
        {   // 16 bytes per lane and 512 per step, the next step's vector in flight: a block's literal area starts at a multiple of
            // 2^17 and has room for the vector that holds its last literal
            const uint4* lit4 = reinterpret_cast<const uint4*>(lit);
            const uint32_t nv = (nlit + 15u) >> 4;
            uint4 cur = lane < nv ? lit4[lane] : make_uint4(0, 0, 0, 0);
            for (uint32_t v0 = 0; v0 < nv; v0 += 32) {
                const uint32_t vi = v0 + lane;
                const uint4 nxt = vi + 32u < nv ? lit4[vi + 32u] : make_uint4(0, 0, 0, 0);
                if (vi < nv) {
                    const uint32_t w[4] = { cur.x, cur.y, cur.z, cur.w };
                    const uint32_t k = nlit - 16u * vi;              // literals left from this vector's first byte
#pragma unroll
                    for (uint32_t j = 0; j < 16; j++)
                        if (j < k) atomicAdd(&ws->hist[(w[j >> 2] >> (8u * (j & 3u))) & 255u], 1u);
                }
                cur = nxt;
            }
        }
        __syncwarp();
        uint32_t ns = 0;
        for (uint32_t i = lane; i < 256; i += 32) ns += ws->hist[i] != 0;
        ns = warp_sum(ns);
        E_TICK(E1C_LITHIST);

        const uint32_t rawHdr = nlit < 32 ? 1u : (nlit < 4096 ? 2u : 3u);
        uint32_t litSecSize = 0;
        bool litDone = false;
        if (nlit >= B2Z_LIT_RLE_MIN && ns == 1) {
            if (lane == 0) {
                if (rawHdr == 1) body[0] = (uint8_t)(1u | (nlit << 3));
                else if (rawHdr == 2) { const uint32_t h = 1u | (1u << 2) | (nlit << 4); body[0] = (uint8_t)h; body[1] = (uint8_t)(h >> 8); }
                else put_hdr3(body, 1u | (3u << 2) | (nlit << 4));
                body[rawHdr] = lit[0];
            }
            litSecSize = rawHdr + 1; litDone = true;
        }
        if (!litDone && nlit >= B2Z_LIT_HUF_MIN && ns >= 2) {
            const bool four = nlit >= 256;
            const uint32_t lh = nlit < 1024 ? 3u : (nlit < 16384 ? 4u : 5u);
            uint32_t maxSym; const uint32_t maxBits = huf_build(ws, lane, &maxSym);
            const uint32_t ts = huf_write_table(ws, body + lh, maxBits, maxSym, lane);
            __syncwarp();
            // exact payload bits from the (unmodified) histogram; decide on the byte bound before writing
            uint32_t T = 0;
            for (uint32_t i = lane; i < 256; i += 32) T += ws->hist[i] * ws->hufLen[i];
            T = warp_sum(T);
            E_TICK(E1C_HUF);
            const uint32_t est = ts + (four ? 6u : 0u) + ((T + 7u) >> 3) + (four ? 4u : 1u);
            if (ts && lh + est < rawHdr + nlit) {
                uint8_t* p = body + lh + ts;
                Stager st;
                uint32_t bodySz;
                if (!four) { st.init(ws->stage, p, lane); bodySz = huf_encode_stream(ws, st, lit, 0, nlit, lane); }
                else {
                    const uint32_t seg = (nlit + 3u) / 4u;
                    st.init(ws->stage, p + 6, lane);
                    const uint32_t s1 = huf_encode_stream(ws, st, lit, 0, seg, lane);
                    const uint32_t s2 = huf_encode_stream(ws, st, lit, seg, 2 * seg, lane);
                    const uint32_t s3 = huf_encode_stream(ws, st, lit, 2 * seg, 3 * seg, lane);
                    const uint32_t s4 = huf_encode_stream(ws, st, lit, 3 * seg, nlit, lane);
                    if (lane == 0) { p[0] = (uint8_t)s1; p[1] = (uint8_t)(s1 >> 8); p[2] = (uint8_t)s2; p[3] = (uint8_t)(s2 >> 8); p[4] = (uint8_t)s3; p[5] = (uint8_t)(s3 >> 8); }
                    bodySz = 6 + s1 + s2 + s3 + s4;
                }
                const uint32_t csize = ts + bodySz;
                if (lane == 0) {
                    const uint32_t sf = !four ? 0u : (lh == 3 ? 1u : (lh == 4 ? 2u : 3u));
                    if (lh == 3) put_hdr3(body, 2u | (sf << 2) | (nlit << 4) | (csize << 14));
                    else if (lh == 4) { const uint32_t h = 2u | (sf << 2) | (nlit << 4) | (csize << 18); body[0] = (uint8_t)h; body[1] = (uint8_t)(h >> 8); body[2] = (uint8_t)(h >> 16); body[3] = (uint8_t)(h >> 24); }
                    else { const uint64_t h = 2ull | (sf << 2) | ((uint64_t)nlit << 4) | ((uint64_t)csize << 22);
                           body[0] = (uint8_t)h; body[1] = (uint8_t)(h >> 8); body[2] = (uint8_t)(h >> 16); body[3] = (uint8_t)(h >> 24); body[4] = (uint8_t)(h >> 32); }
                }
                litSecSize = lh + csize; litDone = true;
            }
        }
        if (!litDone) {                                           // raw literals
            if (lane == 0) {
                if (rawHdr == 1) body[0] = (uint8_t)(nlit << 3);
                else if (rawHdr == 2) { const uint32_t h = (1u << 2) | (nlit << 4); body[0] = (uint8_t)h; body[1] = (uint8_t)(h >> 8); }
                else put_hdr3(body, (3u << 2) | (nlit << 4));
            }
            warp_copy(body + rawHdr, lit, nlit, lane);
            litSecSize = rawHdr + nlit;
        }
        __syncwarp();
        E_TICK(E1C_LITSTREAMS);

        // =========================== sequences section: header and tables
        uint8_t* sp = body + litSecSize;
        uint32_t seqSecSize;
        bool overCap = false;
        {
            uint32_t hdr;
            if (nbSeq < 128) { if (lane == 0) sp[0] = (uint8_t)nbSeq; hdr = 1; }
            else if (nbSeq < 0x7F00) { if (lane == 0) { sp[0] = (uint8_t)((nbSeq >> 8) + 128u); sp[1] = (uint8_t)nbSeq; } hdr = 2; }
            else { if (lane == 0) { sp[0] = 255; sp[1] = (uint8_t)(nbSeq - 0x7F00u); sp[2] = (uint8_t)((nbSeq - 0x7F00u) >> 8); } hdr = 3; }
            seqSecSize = hdr;
        }
        if (nbSeq) {
            uint32_t* cLL = ws->hist; uint32_t* cOF = ws->hist + 64; uint32_t* cML = ws->hist + 128;
            for (uint32_t i = lane; i < 192; i += 32) ws->hist[i] = 0;
            __syncwarp();
            // the three codes of every sequence, LL | OF << 8 | ML << 16, into the block's word area for E2
            uint32_t* codeOut = reinterpret_cast<uint32_t*>(scratch + (size_t)blk * ENT_SCRATCH_STRIDE + sizeof(EntRec));
            uint32_t extra = 0;                                   // sum of raw extra bits (for the size bound)
            uint64_t v[4];                                        // four records per lane, the next four in flight
#pragma unroll
            for (uint32_t m = 0; m < 4; m++) { const uint32_t i = 32u * m + lane; v[m] = i < nbSeq ? sq[i] : 0ull; }
            for (uint32_t i0 = 0; i0 < nbSeq; i0 += 128) {
                uint64_t nx[4];
#pragma unroll
                for (uint32_t m = 0; m < 4; m++) { const uint32_t i = i0 + 128u + 32u * m + lane; nx[m] = i < nbSeq ? sq[i] : 0ull; }
#pragma unroll
                for (uint32_t m = 0; m < 4; m++) {
                    const uint64_t s = v[m];
                    const bool ok = s != 0;                       // past the end: a record is never 0
                    const uint32_t cl = ok ? ll_code(B2Z_SEQ_LL(s)) : 255u, cm = ok ? ml_code(B2Z_SEQ_ML(s) - 3u) : 255u, co = ok ? highbit32(B2Z_SEQ_OFFBASE(s)) : 255u;
                    // one add per distinct code of the 32 (a few codes take most sequences)
                    const uint32_t gl = __match_any_sync(B2Z_FULL, cl), gm = __match_any_sync(B2Z_FULL, cm), go = __match_any_sync(B2Z_FULL, co);
                    if (ok) {
                        codeOut[i0 + 32u * m + lane] = cl | (co << 8) | (cm << 16);
                        if (lane == (uint32_t)__ffs((int)gl) - 1u) atomicAdd(&cLL[cl], (uint32_t)__popc(gl));
                        if (lane == (uint32_t)__ffs((int)gm) - 1u) atomicAdd(&cML[cm], (uint32_t)__popc(gm));
                        if (lane == (uint32_t)__ffs((int)go) - 1u) atomicAdd(&cOF[co], (uint32_t)__popc(go));
                        extra += d_LL_bits[cl] + d_ML_bits[cm] + co;
                    }
                }
#pragma unroll
                for (uint32_t m = 0; m < 4; m++) v[m] = nx[m];
            }
            extra = warp_sum(extra);
            __syncwarp();
            E_TICK(E1C_SEQPASS);
            FseCT* ctL = &ws->u.fse.ct[0]; FseCT* ctO = &ws->u.fse.ct[1]; FseCT* ctM = &ws->u.fse.ct[2];
            uint8_t* tp = sp + seqSecSize + 1;
            uint32_t mL, mO, mM;
            tp += choose_seq_table(ws, ctL, tp, cLL, nbSeq, 35, 9, d_LL_defNorm, 35, 6, &mL, lane);
            tp += choose_seq_table(ws, ctO, tp, cOF, nbSeq, 31, 8, d_OF_defNorm, 28, 5, &mO, lane);
            tp += choose_seq_table(ws, ctM, tp, cML, nbSeq, 52, 9, d_ML_defNorm, 52, 6, &mM, lane);
            if (lane == 0) sp[seqSecSize] = (uint8_t)((mL << 6) | (mO << 4) | (mM << 2));
            seqSecSize += 1 + (uint32_t)(tp - (sp + seqSecSize + 1));
            E_TICK(E1C_TABLES);
            const uint64_t upper = (uint64_t)nbSeq * (ctL->log + ctO->log + ctM->log) + 1ull + extra;
            overCap = (uint64_t)litSecSize + seqSecSize + ((upper + 7ull) >> 3) > B2Z_BODY_CAP;
            if (!overCap) {                                       // hand the tables to E2 and the sizes to E3
                for (uint32_t i = lane; i < ENT_ST_N; i += 32)
                    rec->tab.state[i] = i < ENT_ST_OF ? ctL->state[i] : (i < ENT_ST_ML ? ctO->state[i - ENT_ST_OF] : ctM->state[i - ENT_ST_ML]);
                for (uint32_t i = lane; i < ENT_SY_N; i += 32) {
                    const FseCT* ct = i < ENT_SY_OF ? ctL : (i < ENT_SY_ML ? ctO : ctM);
                    const uint32_t s = i < ENT_SY_OF ? i : (i < ENT_SY_ML ? i - ENT_SY_OF : i - ENT_SY_ML);
                    rec->tab.sym[i] = make_uint2(ct->dnb[s], (uint32_t)ct->dfs[s]);
                }
                if (lane == 0) { rec->run = 1; rec->bodyHead = litSecSize + seqSecSize; rec->logs = ctL->log | (ctO->log << 8) | (ctM->log << 16); }
                __syncwarp();
                E_TICK(E1C_HANDOFF);
                continue;
            }
        }
        __syncwarp();
        const uint32_t outSize = finish_block(out, bsrc, blkSize, last, litSecSize + seqSecSize, overCap, lane);
        if (lane == 0) { slotSize[blk] = outSize; rec->run = 0; }
        __syncwarp();
        E_TICK(E1C_HANDOFF);
    }
    E_CLOCKS_FLUSH(0, E1C_N);
}

// ---------------------------------------------------------------- E2: the FSE state chains, one block per lane
// Lane j of a warp codes block blk0 + j alone: its LL, OF and ML states from the last sequence to the first, three independent
// recurrences in one thread (the serial encoder's order), with the group's tables in the warp's dynamic shared memory.  It reads
// the code words E1 left in the block's word area (LL | OF << 8 | ML << 16), four per 16-byte vector and ENT_CHAIN_VECS vectors
// per round with the next round's in flight, and writes each sequence's state word over its code word: the three states' bits in
// stream order (OF, ML, LL; <= 26 bits) and their count on top.  The last sequence only sets the initial states: its word is 0.
// Lanes without a block to code (E1 finished it, or the group ends) and lanes whose block has run out of sequences idle.
#define ENT_CHAIN_BLOCKS 16                                      // blocks per one-warp CTA, one per lane (lanes 16-31 idle: 4 CTAs
                                                                 // per SM beat 32 blocks and 2 CTAs per SM, DESIGN §2.3)
#define ENT_CHAIN_VECS   4                                       // code vectors per lane per round
#define ENT_CHAIN_SMEM   ((size_t)ENT_CHAIN_BLOCKS * sizeof(EntTables))
__device__ __forceinline__ uint32_t fse_first_state(const uint16_t* stT, uint2 e) {
    const uint32_t nb = (e.x + (1u << 15)) >> 16;
    return stT[(((nb << 16) - e.x) >> nb) + e.y];
}
__device__ __forceinline__ uint32_t fse_step(const uint16_t* stT, uint2 e, uint32_t& state, uint32_t& nbits) {
    nbits = (state + e.x) >> 16;
    const uint32_t bits = state & ((1u << nbits) - 1u);
    state = stT[(state >> nbits) + e.y];
    return bits;
}
__global__ void __launch_bounds__(32)
zstd_enc_chains_kernel(const uint32_t* __restrict__ nseqArr, uint8_t* __restrict__ scratch, uint32_t nBlocks) {
    B2Z_DYN_SMEM(EntTables, tabs);
    const uint32_t lane = threadIdx.x;
    E_CLOCKS_START(E2C_N);
    for (uint32_t blk0 = blockIdx.x * ENT_CHAIN_BLOCKS; blk0 < nBlocks; blk0 += gridDim.x * ENT_CHAIN_BLOCKS) {
        const uint32_t blk = blk0 + lane;
        EntRec* rec = reinterpret_cast<EntRec*>(scratch + (size_t)blk * ENT_SCRATCH_STRIDE);
        const bool mine = lane < ENT_CHAIN_BLOCKS && blk < nBlocks && rec->run;
        const uint32_t n = mine ? nseqArr[blk] : 0u;
        // stage the tables of the group's chained blocks, the whole warp on each (16 bytes per lane per step)
        for (uint32_t run = __ballot_sync(B2Z_FULL, mine); run; run &= run - 1u) {
            const uint32_t j = (uint32_t)__ffs((int)run) - 1u;
            const uint4* s4 = reinterpret_cast<const uint4*>(&reinterpret_cast<const EntRec*>(scratch + (size_t)(blk0 + j) * ENT_SCRATCH_STRIDE)->tab);
            uint4* d4 = reinterpret_cast<uint4*>(&tabs[j]);
            for (uint32_t i = lane; i < sizeof(EntTables) / 16u; i += 32) d4[i] = s4[i];
        }
        __syncwarp();
        E_TICK(E2C_STAGE);
        const EntTables* tb = &tabs[mine ? lane : 0u];
        const uint16_t* stL = tb->state; const uint16_t* stO = tb->state + ENT_ST_OF; const uint16_t* stM = tb->state + ENT_ST_ML;
        const uint2* sy = tb->sym;
        uint4* w4 = reinterpret_cast<uint4*>(scratch + (size_t)(mine ? blk : blk0) * ENT_SCRATCH_STRIDE + sizeof(EntRec));
        const int32_t nV = (int32_t)((n + 3u) >> 2), last = (int32_t)n - 1;
        const uint32_t rounds = warp_max(((uint32_t)nV + ENT_CHAIN_VECS - 1u) / ENT_CHAIN_VECS);
        uint4 cur[ENT_CHAIN_VECS];
#pragma unroll
        for (int32_t m = 0; m < ENT_CHAIN_VECS; m++) { const int32_t q = nV - 1 - m; cur[m] = q >= 0 ? w4[q] : make_uint4(0, 0, 0, 0); }
        uint32_t sL = 0, sO = 0, sM = 0;
        if (n) {                                                 // the last sequence sets the initial states
            const uint32_t e = (uint32_t)last & 3u;
            const uint32_t c = e == 0 ? cur[0].x : (e == 1 ? cur[0].y : (e == 2 ? cur[0].z : cur[0].w));
            sL = fse_first_state(stL, sy[c & 255u]);
            sO = fse_first_state(stO, sy[ENT_SY_OF + ((c >> 8) & 255u)]);
            sM = fse_first_state(stM, sy[ENT_SY_ML + (c >> 16)]);
        }
        E_TICK(E2C_LOAD);
        for (uint32_t r = 0; r < rounds; r++) {
            const int32_t q0 = nV - 1 - (int32_t)(r * ENT_CHAIN_VECS);
            uint4 nxt[ENT_CHAIN_VECS];
#pragma unroll
            for (int32_t m = 0; m < ENT_CHAIN_VECS; m++) {
                const int32_t q = q0 - ENT_CHAIN_VECS - m;
                nxt[m] = q >= 0 ? w4[q] : make_uint4(0, 0, 0, 0);
            }
            E_TICK(E2C_LOAD);
#pragma unroll
            for (int32_t m = 0; m < ENT_CHAIN_VECS; m++) {
                const int32_t q = q0 - m;
                if (q < 0) continue;
                uint32_t w[4] = { cur[m].x, cur[m].y, cur[m].z, cur[m].w };
#pragma unroll
                for (int32_t e = 3; e >= 0; e--) {
                    const int32_t i = 4 * q + e;
                    if (i < last) {
                        const uint32_t c = w[e];
                        const uint2 eL = sy[c & 255u], eO = sy[ENT_SY_OF + ((c >> 8) & 255u)], eM = sy[ENT_SY_ML + (c >> 16)];
                        uint32_t nL, nO, nM;
                        const uint32_t bO = fse_step(stO, eO, sO, nO), bM = fse_step(stM, eM, sM, nM), bL = fse_step(stL, eL, sL, nL);
                        w[e] = bO | (bM << nO) | (bL << (nO + nM)) | ((nO + nM + nL) << 26);
                    } else if (i == last) {
                        w[e] = 0;
                    }
                }
                cur[m] = make_uint4(w[0], w[1], w[2], w[3]);
            }
            E_TICK(E2C_STEP);
#pragma unroll
            for (int32_t m = 0; m < ENT_CHAIN_VECS; m++) {
                const int32_t q = q0 - m;
                if (q >= 0) w4[q] = cur[m];
                cur[m] = nxt[m];
            }
            E_TICK(E2C_STORE);
        }
        if (n) { rec->fin[0] = (uint16_t)sL; rec->fin[1] = (uint16_t)sO; rec->fin[2] = (uint16_t)sM; }
        __syncwarp();
        E_TICK(E2C_STORE);
    }
    E_CLOCKS_FLUSH(E1C_N, E2C_N);
}

// ---------------------------------------------------------------- E3: the sequence bitstream, one warp per block
__global__ void __launch_bounds__(B2Z_ENT_WARPS * 32)
zstd_enc_seqbits_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g,
                        const uint64_t* __restrict__ seqs, const uint32_t* __restrict__ nseqArr,
                        uint8_t* __restrict__ slots, uint32_t* __restrict__ slotSize, const uint8_t* __restrict__ scratch, uint32_t nBlocks) {
    __shared__ uint32_t stageAll[B2Z_ENT_WARPS][STAGE_WORDS];
    const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
    for (uint32_t blk = blockIdx.x * B2Z_ENT_WARPS + wib; blk < nBlocks; blk += gridDim.x * B2Z_ENT_WARPS) {
        const EntRec* rec = reinterpret_cast<const EntRec*>(scratch + (size_t)blk * ENT_SCRATCH_STRIDE);
        if (!rec->run) continue;
        const uint32_t* words = reinterpret_cast<const uint32_t*>(scratch + (size_t)blk * ENT_SCRATCH_STRIDE + sizeof(EntRec));
        const BlockGeom bg = block_geom(g, srcSize, blk);
        const uint64_t* sq = seqs + (size_t)blk * B2Z_MAXSEQ;
        const uint32_t nbSeq = nseqArr[blk], bodyHead = rec->bodyHead, logs = rec->logs;
        const uint32_t logL = logs & 255u, logO = (logs >> 8) & 255u, logM = logs >> 16;
        uint8_t* out = slots + (size_t)blk * B2Z_SLOT;
        Stager st; st.init(stageAll[wib], out + 3 + bodyHead, lane);
        uint8_t* bsStart = st.out;
        // sequences walked last -> first, 32 per step: state bits (OF, ML, LL), then LL, ML, OF extra bits
        for (uint32_t hi = nbSeq; hi > 0;) {
            const uint32_t cnt = hi < 32u ? hi : 32u;
            uint64_t lo = 0; uint32_t hiw = 0, nb = 0;
            if (lane < cnt) {
                const uint32_t i = hi - 1u - lane;
                const uint64_t s = sq[i]; const uint32_t w = words[i];
                const uint32_t llv = B2Z_SEQ_LL(s), mlv = B2Z_SEQ_ML(s), obv = B2Z_SEQ_OFFBASE(s);
                const uint32_t cl = ll_code(llv), cm = ml_code(mlv - 3u), co = highbit32(obv);
                lo = w & 0x3FFFFFFu; nb = w >> 26;                                     // <= 26 bits
                const uint32_t lb = d_LL_bits[cl], mb = d_ML_bits[cm];
                lo |= (uint64_t)(llv - d_LL_base[cl]) << nb; nb += lb;                 // <= 42
                lo |= (uint64_t)(mlv - d_ML_base[cm]) << nb; nb += mb;                 // <= 58
                const uint32_t ox = obv - (1u << co);
                if (nb + co <= 64) { lo |= (co ? ((uint64_t)ox << nb) : 0ull); }
                else { lo |= (uint64_t)ox << nb; hiw = (uint32_t)((uint64_t)ox >> (64u - nb)); }
                nb += co;
            }
            uint32_t total; const uint32_t off = warp_excl_scan(nb, lane, &total);
            st.put(st.bits + off, lo, hiw, nb);
            st.bits += total; hi -= cnt;
            if (st.bits > STAGE_FLUSH_BITS) st.flush(lane, false);
        }
        // final states: ML, OF, LL, then end mark
        if (lane == 0) {
            uint32_t o = st.bits;
            st.put(o, rec->fin[2] & ((1u << logM) - 1u), 0, logM); o += logM;
            st.put(o, rec->fin[1] & ((1u << logO) - 1u), 0, logO); o += logO;
            st.put(o, rec->fin[0] & ((1u << logL) - 1u), 0, logL); o += logL;
            st.put(o, 1, 0, 1);
        }
        st.bits += logM + logO + logL + 1u;
        st.flush(lane, true);
        const uint32_t bodySize = bodyHead + (uint32_t)(st.out - bsStart);
        const uint32_t outSize = finish_block(out, src + bg.litOff, bg.blkSize, bg.last, bodySize, false, lane);
        if (lane == 0) slotSize[blk] = outSize;
        __syncwarp();
    }
}

#ifndef B2Z_CUEMU
#ifdef B2Z_E_CLOCKS
// the per-phase cycle sums of the E1 and E2 warps since the last call (E1C_* order, then E2C_*); clears them
extern "C" int b200z_e_clocks(unsigned long long* out) {
    static const unsigned long long zero[E1C_N + E2C_N] = {};
    cudaError_t e = cudaMemcpyFromSymbol(out, e_clocks, sizeof(e_clocks));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(e_clocks, zero, sizeof(e_clocks));
    return (int)e;
}
#endif
void launch_zstd_enc_entropy(const uint8_t* src, uint64_t srcSize, const EncGeom& g,
                             const uint64_t* seqs, const uint32_t* nseq, const uint8_t* lits, const uint32_t* nlit,
                             uint8_t* slots, uint32_t* slotSize, uint8_t* scratch, uint32_t nBlocks, uint32_t smCount, cudaStream_t st) {
    if (!nBlocks) return;
    uint32_t grid = (nBlocks + B2Z_ENT_WARPS - 1) / B2Z_ENT_WARPS;
    const uint32_t cap = smCount * 16u;
    if (grid > cap) grid = cap;
    zstd_enc_tables_kernel<<<grid, B2Z_ENT_WARPS * 32, 0, st>>>(src, srcSize, g, seqs, nseq, lits, nlit, slots, slotSize, scratch, nBlocks);
    cudaFuncSetAttribute(zstd_enc_chains_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ENT_CHAIN_SMEM);
    cudaFuncSetAttribute(zstd_enc_chains_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    zstd_enc_chains_kernel<<<(nBlocks + ENT_CHAIN_BLOCKS - 1) / ENT_CHAIN_BLOCKS, 32, ENT_CHAIN_SMEM, st>>>(nseq, scratch, nBlocks);
    zstd_enc_seqbits_kernel<<<grid, B2Z_ENT_WARPS * 32, 0, st>>>(src, srcSize, g, seqs, nseq, slots, slotSize, scratch, nBlocks);
}
#else
// Host emulation (tests/cuemu): the emulator's stage E entry launches zstd_enc_entropy_kernel once, over 4-warp CTAs of the
// blocks.  Stage E is three launches with scratch between them, so under the emulator that entry's first thread runs E1, E2
// and E3 in turn over every block -- the launches launch_zstd_enc_entropy makes, E2 as one-warp CTAs of ENT_CHAIN_BLOCKS blocks
// with ENT_CHAIN_SMEM bytes of dynamic shared memory -- with scratch of its own, and counts their collectives as its own.  Every
// other thread returns at once.
inline void zstd_enc_entropy_kernel(const uint8_t* src, uint64_t srcSize, EncGeom g, const uint64_t* seqs, const uint32_t* nseq,
                                    const uint8_t* lits, const uint32_t* nlit, uint8_t* slots, uint32_t* slotSize, uint32_t nBlocks) {
    if (blockIdx.x != 0 || threadIdx.x != 0 || !nBlocks) return;
    cuemu::Block* const outer = cuemu::blk();
    std::vector<uint8_t> buf((size_t)nBlocks * ENT_SCRATCH_STRIDE + 16, 0xCD);
    uint8_t* const scratch = buf.data() + ((16u - ((uintptr_t)buf.data() & 15u)) & 15u);
    const dim3 grid((nBlocks + B2Z_ENT_WARPS - 1) / B2Z_ENT_WARPS), block(B2Z_ENT_WARPS * 32);
    uint64_t c = cuemu::launch(grid, block, 0, [&] { zstd_enc_tables_kernel(src, srcSize, g, seqs, nseq, lits, nlit, slots, slotSize, scratch, nBlocks); });
    c += cuemu::launch(dim3((nBlocks + ENT_CHAIN_BLOCKS - 1) / ENT_CHAIN_BLOCKS), dim3(32), ENT_CHAIN_SMEM, [&] { zstd_enc_chains_kernel(nseq, scratch, nBlocks); });
    c += cuemu::launch(grid, block, 0, [&] { zstd_enc_seqbits_kernel(src, srcSize, g, seqs, nseq, slots, slotSize, scratch, nBlocks); });
    cuemu::blk() = outer;                                        // each launch leaves the emulator without a current CTA
    outer->collectives += c;
}
#endif

}  // namespace b2z
