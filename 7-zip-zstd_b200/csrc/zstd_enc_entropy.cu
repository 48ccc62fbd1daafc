// zstd_enc_entropy.cu -- stage E of the block-parallel Zstandard encoder (sm_90a).
//
// One WARP compresses one 128 KiB block from stage M's output (final sequences + literal
// bytes) into a complete zstd block (3-byte header + literals section + sequences section)
// written to the block's slot.  All 32 lanes cooperate on the data-parallel parts:
//   - byte histogram of the literals (shared-memory atomics),
//   - Huffman bit-packing of the 4 literal streams: 32 symbols per iteration, bit offsets by
//     warp-shuffle prefix sums, codes OR-ed into a shared-memory staging window,
//   - code histograms of the sequences, and the bit assembly of the sequence stream
//     (per sequence: three FSE state emissions + LL/ML/OF extra bits).
// The inherently serial chains run on single lanes while many warps are in flight:
//   - Huffman tree construction, table descriptions, FSE normalisation/table build (lane 0),
//   - the three FSE state chains (lanes 0,1,2 -- one per symbol type).
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

__device__ __forceinline__ uint32_t ll_code(uint32_t ll) {
    if (ll < 16) return ll;
    if (ll < 24) return 16 + ((ll - 16) >> 1);
    if (ll < 32) return 20 + ((ll - 24) >> 2);
    if (ll < 48) return 22 + ((ll - 32) >> 3);
    if (ll < 64) return 24;
    return highbit32(ll) + 19;
}
__device__ __forceinline__ uint32_t ml_code(uint32_t m) {   // m = matchLength - 3
    if (m < 32) return m;
    if (m < 40) return 32 + ((m - 32) >> 1);
    if (m < 48) return 36 + ((m - 40) >> 2);
    if (m < 64) return 38 + ((m - 48) >> 3);
    if (m < 96) return 40 + ((m - 64) >> 4);
    if (m < 128) return 42;
    return highbit32(m) + 36;
}

// ---------------------------------------------------------------- per-warp workspace
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
        struct { uint32_t w[512]; uint16_t parent[512]; uint8_t order[256]; uint8_t depth[512]; } hb;   // Huffman build
        struct { FseCT ct[3]; } fse;                                                                      // LL, OF, ML
    } u;
    uint8_t  spread[512];            // FSE symbol spreading scratch
    int16_t  norm[64];
    uint32_t stage[STAGE_WORDS];     // bit staging window
    uint8_t  bcode[3][32];           // per-batch codes (LL, OF, ML)
    uint16_t bbits[3][32];           // per-batch FSE state bits
    uint8_t  bnb[3][32];
};

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

// ---------------------------------------------------------------- FSE (lane 0)
__device__ void fse_build_ctable(FseCT* ct, uint8_t* spread, const int16_t* norm, uint32_t maxSym, uint32_t log) {
    const uint32_t size = 1u << log, mask = size - 1u, step = (size >> 1) + (size >> 3) + 3u;
    uint32_t cumul[65], high = size - 1u;
    cumul[0] = 0;
    for (uint32_t s = 0; s <= maxSym; s++) {
        if (norm[s] == -1) { cumul[s + 1] = cumul[s] + 1u; spread[high--] = (uint8_t)s; }
        else cumul[s + 1] = cumul[s] + (uint32_t)norm[s];
    }
    uint32_t pos = 0;
    for (uint32_t s = 0; s <= maxSym; s++)
        for (int i = 0; i < norm[s]; i++) { spread[pos] = (uint8_t)s; pos = (pos + step) & mask; while (pos > high) pos = (pos + step) & mask; }
    for (uint32_t u = 0; u < size; u++) { const uint32_t s = spread[u]; ct->state[cumul[s]++] = (uint16_t)(size + u); }
    uint32_t total = 0;
    for (uint32_t s = 0; s <= maxSym; s++) {
        const int n = norm[s];
        if (n == 0) { ct->dnb[s] = ((log + 1u) << 16) - size; ct->dfs[s] = 0; }
        else if (n == 1 || n == -1) { ct->dnb[s] = (log << 16) - size; ct->dfs[s] = (int32_t)total - 1; total++; }
        else {
            const uint32_t maxBitsOut = log - highbit32((uint32_t)n - 1u), minStatePlus = (uint32_t)n << maxBitsOut;
            ct->dnb[s] = (maxBitsOut << 16) - minStatePlus;
            ct->dfs[s] = (int32_t)total - n; total += (uint32_t)n;
        }
    }
    ct->log = log;
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

__device__ void fse_normalize(int16_t* norm, uint32_t log, const uint32_t* count, uint32_t total, uint32_t maxSym) {
    const uint32_t size = 1u << log; int32_t sum = 0;
    for (uint32_t s = 0; s <= maxSym; s++) {
        if (!count[s]) { norm[s] = 0; continue; }
        uint64_t p = ((uint64_t)count[s] * size * 2u + total) / (2ull * total);
        if (p < 1) p = 1;
        norm[s] = (int16_t)p; sum += (int32_t)p;
    }
    int32_t delta = (int32_t)size - sum;
    while (delta != 0) {
        uint32_t big = 0;
        for (uint32_t s = 1; s <= maxSym; s++) if (norm[s] > norm[big]) big = s;
        if (delta > 0) { norm[big] = (int16_t)(norm[big] + delta); delta = 0; }
        else {
            int32_t take = norm[big] - 1 < -delta ? norm[big] - 1 : -delta;
            if (take > (norm[big] >> 1) && norm[big] > 2) take = norm[big] >> 1;
            norm[big] = (int16_t)(norm[big] - take); delta += take;
        }
    }
}

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
__device__ uint64_t fse_cost_fx8(const uint32_t* count, const int16_t* norm, uint32_t maxSym, uint32_t log) {
    uint64_t c = 0;
    for (uint32_t s = 0; s <= maxSym; s++) {
        if (!count[s]) continue;
        if (norm[s] == 0) return ~0ull;
        const uint32_t n = norm[s] < 0 ? 1u : (uint32_t)norm[s];
        c += (uint64_t)count[s] * ((log << 8) - log2_fx8(n));
    }
    return c;
}

// ---------------------------------------------------------------- Huffman (lane 0)
// code lengths (<= 11) into ws->hufLen / hufCode; returns maxBits, sets *maxSymOut
__device__ uint32_t huf_build(WarpWS* ws, uint32_t* maxSymOut) {
    uint32_t* count = ws->hist;
    uint32_t* w = ws->u.hb.w; uint16_t* parent = ws->u.hb.parent; uint8_t* order = ws->u.hb.order; uint8_t* depth = ws->u.hb.depth;
    uint32_t n, maxd;
#define EFFC(s) ((count[s] + (1u << k) - 1u) >> k)          /* count after k halvings (ceil) */
    for (uint32_t k = 0;; k++) {
        n = 0;
        for (uint32_t s = 0; s < 256; s++) if (count[s]) order[n++] = (uint8_t)s;
        for (uint32_t i = 1; i < n; i++) {                       // stable insertion sort by count
            const uint32_t s = order[i], c = EFFC(s); int j = (int)i - 1;
            while (j >= 0 && EFFC(order[j]) > c) { order[j + 1] = order[j]; j--; }
            order[j + 1] = (uint8_t)s;
        }
        for (uint32_t i = 0; i < n; i++) w[i] = EFFC(order[i]);
        uint32_t li = 0, ii = n, ie = n;
        while ((n - li) + (ie - ii) > 1) {
            uint32_t a, b;
            if (li < n && (ii >= ie || w[li] <= w[ii])) a = li++; else a = ii++;
            if (li < n && (ii >= ie || w[li] <= w[ii])) b = li++; else b = ii++;
            w[ie] = w[a] + w[b]; parent[a] = (uint16_t)ie; parent[b] = (uint16_t)ie; ie++;
        }
        maxd = 0; depth[ie - 1] = 0;
        for (int i = (int)ie - 2; i >= 0; i--) depth[i] = (uint8_t)(depth[parent[i]] + 1);
        for (uint32_t i = 0; i < n; i++) if (depth[i] > maxd) maxd = depth[i];
        if (maxd <= 11) break;
    }
#undef EFFC
    for (uint32_t s = 0; s < 256; s++) ws->hufLen[s] = 0;
    for (uint32_t i = 0; i < n; i++) ws->hufLen[order[i]] = depth[i];
    uint32_t maxSym = 0;
    for (uint32_t s = 0; s < 256; s++) if (count[s]) maxSym = s;
    uint32_t rank[13], start[13], pos = 0;
    for (uint32_t r = 0; r < 13; r++) rank[r] = 0;
    for (uint32_t s = 0; s < 256; s++) if (ws->hufLen[s]) rank[maxd + 1u - ws->hufLen[s]]++;
    for (uint32_t r = 1; r <= maxd; r++) { start[r] = pos; pos += rank[r] << (r - 1u); }
    for (uint32_t s = 0; s < 256; s++) {
        if (!ws->hufLen[s]) { ws->hufCode[s] = 0; continue; }
        const uint32_t r = maxd + 1u - ws->hufLen[s];
        ws->hufCode[s] = (uint16_t)(start[r] >> (r - 1u)); start[r] += 1u << (r - 1u);
    }
    *maxSymOut = maxSym;
    return maxd;
}

// tree description at dst; returns bytes written or 0 (not representable)
__device__ uint32_t huf_write_table(WarpWS* ws, uint8_t* dst, uint32_t maxBits, uint32_t maxSym) {
    const uint32_t nw = maxSym;
    uint8_t* wt = ws->u.hb.order;                                // weights (hb scratch is dead now; order[256] reused)
    for (uint32_t s = 0; s < nw; s++) wt[s] = ws->hufLen[s] ? (uint8_t)(maxBits + 1u - ws->hufLen[s]) : 0;
    uint32_t fseSize = 0;
    if (nw > 1) {
        uint32_t cnt[16], maxW = 0, maxCnt = 0;
        for (uint32_t i = 0; i < 16; i++) cnt[i] = 0;
        for (uint32_t i = 0; i < nw; i++) { cnt[wt[i]]++; if (wt[i] > maxW) maxW = wt[i]; }
        for (uint32_t i = 0; i <= maxW; i++) if (cnt[i] > maxCnt) maxCnt = cnt[i];
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
            fse_normalize(norm, log, cnt, nw, maxW);
            uint8_t* tmp = dst + 1;
            const uint32_t hs = fse_write_ncount(tmp, norm, maxW, log);
            // weights table: a 64-state FseCT carved out of the stage buffer (unused at this point)
            FseCT* ct = reinterpret_cast<FseCT*>(ws->u.hb.w);    // hb.w (2 KiB) + parent: large enough for FseCT? see static_assert
            fse_build_ctable(ct, ws->spread, norm, maxW, log);
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
    }
    const uint32_t rawSize = (nw + 1u) / 2u;
    if (fseSize && fseSize < 128u && (fseSize < rawSize || nw > 128u)) { dst[0] = (uint8_t)fseSize; return 1u + fseSize; }
    if (nw > 128u || nw == 0u) return 0;
    dst[0] = (uint8_t)(127u + nw);
    for (uint32_t i = 0; i < nw; i += 2) dst[1 + i / 2] = (uint8_t)((wt[i] << 4) | (i + 1 < nw ? wt[i + 1] : 0));
    return 1u + rawSize;
}
static_assert(sizeof(FseCT) <= sizeof(uint32_t) * 512 + sizeof(uint16_t) * 512, "weights FseCT must fit in hb.w+hb.parent");

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

// Huffman-encode literals [a, b) as one backward stream at st.out; returns stream bytes
__device__ uint32_t huf_encode_stream(WarpWS* ws, Stager& st, const uint8_t* __restrict__ lit, uint32_t a, uint32_t b, uint32_t lane) {
    uint8_t* start = st.out;
    for (uint32_t hi = b; hi > a;) {
        const uint32_t cnt = (hi - a) < 32u ? (hi - a) : 32u;
        uint32_t code = 0, nb = 0;
        if (lane < cnt) { const uint32_t s = lit[hi - 1u - lane]; code = ws->hufCode[s]; nb = ws->hufLen[s]; }
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

// ---------------------------------------------------------------- sequence table choice (lane 0)
// returns header bytes written at dst; *mode = 0 predefined, 1 RLE, 2 compressed
__device__ uint32_t choose_seq_table(WarpWS* ws, FseCT* ct, uint8_t* dst, const uint32_t* count, uint32_t nbSeq, uint32_t maxSymAll,
                                     uint32_t maxLog, const int16_t* defNorm, uint32_t defMaxSym, uint32_t defLog, uint32_t* mode) {
    uint32_t maxSym = 0, present = 0, big = 0;
    for (uint32_t s = 0; s <= maxSymAll; s++) if (count[s]) { maxSym = s; present++; if (count[s] > big) big = count[s]; }
    if (big == nbSeq && !(nbSeq <= 2 && maxSym <= defMaxSym)) {
        for (uint32_t s = 0; s < 64; s++) { ct->dnb[s] = 0; ct->dfs[s] = 0; }
        ct->state[0] = 0; ct->state[1] = 0; ct->log = 0;
        *mode = 1; dst[0] = (uint8_t)maxSym; return 1;
    }
    int16_t* norm = ws->norm;
    // default-table cost (copy default norm into smem for the shared cost routine)
    uint64_t costDef = ~0ull;
    if (maxSym <= defMaxSym) { for (uint32_t s = 0; s <= defMaxSym; s++) norm[s] = defNorm[s]; costDef = fse_cost_fx8(count, norm, maxSym, defLog); }
    const uint32_t hbN = highbit32(nbSeq > 1 ? nbSeq - 1u : 1u);
    uint32_t log = hbN >= 2 ? hbN - 2u : 0u;
    const uint32_t minA = highbit32(nbSeq) + 1u, minB = highbit32(maxSym ? maxSym : 1u) + 2u, lo = minA < minB ? minA : minB;
    if (log > maxLog) log = maxLog;
    if (log < lo) log = lo;
    if (log < 5) log = 5;
    if (log > maxLog) log = maxLog;
    while ((1u << log) < present) log++;
    fse_normalize(norm, log, count, nbSeq, maxSym);
    const uint32_t hs = fse_write_ncount(dst, norm, maxSym, log);
    const uint64_t costFse = fse_cost_fx8(count, norm, maxSym, log) + ((uint64_t)hs << 11);
    if (costDef <= costFse || big == nbSeq) {
        for (uint32_t s = 0; s <= defMaxSym; s++) norm[s] = defNorm[s];
        fse_build_ctable(ct, ws->spread, norm, defMaxSym, defLog); *mode = 0; return 0;
    }
    fse_build_ctable(ct, ws->spread, norm, maxSym, log); *mode = 2; return hs;
}

// ---------------------------------------------------------------- the kernel
__global__ void __launch_bounds__(B2Z_ENT_WARPS * 32)
zstd_enc_entropy_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g,
                        const uint64_t* __restrict__ seqs, const uint32_t* __restrict__ nseqArr,
                        const uint8_t* __restrict__ lits, const uint32_t* __restrict__ nlitArr,
                        uint8_t* __restrict__ slots, uint32_t* __restrict__ slotSize, uint32_t nBlocks) {
    __shared__ WarpWS wsAll[B2Z_ENT_WARPS];
    const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
    WarpWS* ws = &wsAll[wib];
    const uint32_t blocksPerFrame = 1u << (g.frameLog - 17u);
    for (uint32_t blk = blockIdx.x * B2Z_ENT_WARPS + wib; blk < nBlocks; blk += gridDim.x * B2Z_ENT_WARPS) {
        // geometry of this block
        const uint64_t frame = blk / blocksPerFrame; const uint32_t bif = blk % blocksPerFrame;
        const uint64_t f0 = frame << g.frameLog;
        const uint64_t fn = enc_frame_bytes(g, srcSize, frame);
        const uint64_t b0 = (uint64_t)bif << 17;
        const uint32_t blkSize = (uint32_t)((fn - b0) < B2Z_BLOCK ? (fn - b0) : B2Z_BLOCK);
        const uint32_t last = (b0 + blkSize == fn) ? 1u : 0u;
        const uint8_t* bsrc = src + f0 + b0;
        const uint8_t* lit = lits + f0 + b0;
        const uint64_t* sq = seqs + (size_t)blk * B2Z_MAXSEQ;
        const uint32_t nbSeq = nseqArr[blk], nlit = nlitArr[blk];
        uint8_t* out = slots + (size_t)blk * B2Z_SLOT;
        uint8_t* body = out + 3;
        uint32_t outSize;

        // RLE block?
        bool rle = false;
        if (blkSize > 1 && nbSeq == 1 && nlit == 1) {
            const uint64_t s0 = sq[0];
            rle = B2Z_SEQ_LL(s0) == 1 && B2Z_SEQ_ML(s0) == blkSize - 1u && B2Z_SEQ_OFFBASE(s0) == 4u;
        }
        if (rle) {
            if (lane == 0) { const uint32_t h = last | (1u << 1) | (blkSize << 3); out[0] = (uint8_t)h; out[1] = (uint8_t)(h >> 8); out[2] = (uint8_t)(h >> 16); out[3] = bsrc[0]; slotSize[blk] = 4; }
            continue;
        }

        // =========================== literals section
        for (uint32_t i = lane; i < 256; i += 32) ws->hist[i] = 0;
        __syncwarp();
        for (uint32_t i = lane * 4; i < nlit; i += 128) {
            const uint32_t v = *reinterpret_cast<const uint32_t*>(lit + i);   // block literal area is 4-byte aligned, in-bounds (<= blkSize rounded)
            const uint32_t k = nlit - i;
            atomicAdd(&ws->hist[v & 255u], 1u);
            if (k > 1) atomicAdd(&ws->hist[(v >> 8) & 255u], 1u);
            if (k > 2) atomicAdd(&ws->hist[(v >> 16) & 255u], 1u);
            if (k > 3) atomicAdd(&ws->hist[v >> 24], 1u);
        }
        __syncwarp();
        uint32_t ns = 0;
        for (uint32_t i = lane; i < 256; i += 32) ns += ws->hist[i] != 0;
        for (int d = 16; d; d >>= 1) ns += __shfl_xor_sync(B2Z_FULL, ns, d);

        const uint32_t rawHdr = nlit < 32 ? 1u : (nlit < 4096 ? 2u : 3u);
        uint32_t litSecSize = 0;
        bool litDone = false;
        if (nlit >= B2Z_LIT_RLE_MIN && ns == 1) {
            if (lane == 0) {
                if (rawHdr == 1) body[0] = (uint8_t)(1u | (nlit << 3));
                else if (rawHdr == 2) { const uint32_t h = 1u | (1u << 2) | (nlit << 4); body[0] = (uint8_t)h; body[1] = (uint8_t)(h >> 8); }
                else { const uint32_t h = 1u | (3u << 2) | (nlit << 4); body[0] = (uint8_t)h; body[1] = (uint8_t)(h >> 8); body[2] = (uint8_t)(h >> 16); }
                body[rawHdr] = lit[0];
            }
            litSecSize = rawHdr + 1; litDone = true;
        }
        if (!litDone && nlit >= B2Z_LIT_HUF_MIN && ns >= 2) {
            const bool four = nlit >= 256;
            const uint32_t lh = nlit < 1024 ? 3u : (nlit < 16384 ? 4u : 5u);
            uint32_t ts = 0;
            if (lane == 0) {
                uint32_t maxSym; const uint32_t maxBits = huf_build(ws, &maxSym);
                ts = huf_write_table(ws, body + lh, maxBits, maxSym);
            }
            ts = __shfl_sync(B2Z_FULL, ts, 0);
            __syncwarp();
            // exact payload bits from the (unmodified) histogram; decide on the byte bound before writing
            uint32_t T = 0;
            for (uint32_t i = lane; i < 256; i += 32) T += ws->hist[i] * ws->hufLen[i];
            for (int d = 16; d; d >>= 1) T += __shfl_xor_sync(B2Z_FULL, T, d);
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
                    if (lh == 3) { const uint32_t h = 2u | (sf << 2) | (nlit << 4) | (csize << 14); body[0] = (uint8_t)h; body[1] = (uint8_t)(h >> 8); body[2] = (uint8_t)(h >> 16); }
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
                else { const uint32_t h = (3u << 2) | (nlit << 4); body[0] = (uint8_t)h; body[1] = (uint8_t)(h >> 8); body[2] = (uint8_t)(h >> 16); }
            }
            warp_copy(body + rawHdr, lit, nlit, lane);
            litSecSize = rawHdr + nlit;
        }
        __syncwarp();

        // =========================== sequences section
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
            uint32_t extra = 0;                                   // sum of raw extra bits (for the size bound)
            for (uint32_t i = lane; i < nbSeq; i += 32) {
                const uint64_t s = sq[i];
                const uint32_t cl = ll_code(B2Z_SEQ_LL(s)), cm = ml_code(B2Z_SEQ_ML(s) - 3u), co = highbit32(B2Z_SEQ_OFFBASE(s));
                atomicAdd(&cLL[cl], 1u); atomicAdd(&cML[cm], 1u); atomicAdd(&cOF[co], 1u);
                extra += d_LL_bits[cl] + d_ML_bits[cm] + co;
            }
            for (int d = 16; d; d >>= 1) extra += __shfl_xor_sync(B2Z_FULL, extra, d);
            __syncwarp();
            FseCT* ctL = &ws->u.fse.ct[0]; FseCT* ctO = &ws->u.fse.ct[1]; FseCT* ctM = &ws->u.fse.ct[2];
            uint32_t tblBytes = 0;
            if (lane == 0) {
                uint8_t* tp = sp + seqSecSize + 1;
                uint32_t mL, mO, mM;
                tp += choose_seq_table(ws, ctL, tp, cLL, nbSeq, 35, 9, d_LL_defNorm, 35, 6, &mL);
                tp += choose_seq_table(ws, ctO, tp, cOF, nbSeq, 31, 8, d_OF_defNorm, 28, 5, &mO);
                tp += choose_seq_table(ws, ctM, tp, cML, nbSeq, 52, 9, d_ML_defNorm, 52, 6, &mM);
                sp[seqSecSize] = (uint8_t)((mL << 6) | (mO << 4) | (mM << 2));
                tblBytes = (uint32_t)(tp - (sp + seqSecSize + 1));
            }
            tblBytes = __shfl_sync(B2Z_FULL, tblBytes, 0);
            __syncwarp();
            seqSecSize += 1 + tblBytes;
            {
                const uint64_t upper = (uint64_t)nbSeq * (ctL->log + ctO->log + ctM->log) + 1ull + extra;
                overCap = (uint64_t)litSecSize + seqSecSize + ((upper + 7ull) >> 3) > B2Z_BODY_CAP;
            }
            if (!overCap) {
            // ---- bitstream: sequences walked last -> first, 32 per batch
            Stager st; st.init(ws->stage, sp + seqSecSize, lane);
            uint8_t* bsStart = st.out;
            uint32_t stL = 0, stO = 0, stM = 0;                   // chain states: valid on lanes 0,1,2
            bool first = true;
            for (uint32_t hi = nbSeq; hi > 0;) {
                const uint32_t cnt = hi < 32u ? hi : 32u;
                uint32_t llv = 0, mlv = 0, obv = 1, cl = 0, cm = 0, co = 0;
                if (lane < cnt) {
                    const uint64_t s = sq[hi - 1u - lane];
                    llv = B2Z_SEQ_LL(s); mlv = B2Z_SEQ_ML(s); obv = B2Z_SEQ_OFFBASE(s);
                    cl = ll_code(llv); cm = ml_code(mlv - 3u); co = highbit32(obv);
                    ws->bcode[0][lane] = (uint8_t)cl; ws->bcode[1][lane] = (uint8_t)co; ws->bcode[2][lane] = (uint8_t)cm;
                }
                __syncwarp();
                if (lane < 3) {                                   // the three FSE chains
                    const FseCT* ct = lane == 0 ? ctL : (lane == 1 ? ctO : ctM);
                    uint32_t state = lane == 0 ? stL : (lane == 1 ? stO : stM);
                    uint32_t k = 0;
                    if (first) { state = fse_init_state(ct, ws->bcode[lane][0]); ws->bbits[lane][0] = 0; ws->bnb[lane][0] = 0; k = 1; }
                    for (; k < cnt; k++) {
                        uint32_t nb; const uint32_t bits = fse_encode(ct, &state, ws->bcode[lane][k], &nb);
                        ws->bbits[lane][k] = (uint16_t)bits; ws->bnb[lane][k] = (uint8_t)nb;
                    }
                    if (lane == 0) stL = state; else if (lane == 1) stO = state; else stM = state;
                }
                __syncwarp();
                // assemble: OF state, ML state, LL state, then LL, ML, OF extra bits
                uint64_t lo = 0; uint32_t hiw = 0, nb = 0;
                if (lane < cnt) {
                    const uint32_t nO = ws->bnb[1][lane], nM = ws->bnb[2][lane], nL = ws->bnb[0][lane];
                    lo = ws->bbits[1][lane]; nb = nO;
                    lo |= (uint64_t)ws->bbits[2][lane] << nb; nb += nM;
                    lo |= (uint64_t)ws->bbits[0][lane] << nb; nb += nL;                  // <= 26 bits
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
                st.bits += total; hi -= cnt; first = false;
                if (st.bits > STAGE_FLUSH_BITS) st.flush(lane, false);
            }
            // final states: ML, OF, LL, then end mark
            {
                const uint32_t sM = __shfl_sync(B2Z_FULL, stM, 2), sO = __shfl_sync(B2Z_FULL, stO, 1), sL = __shfl_sync(B2Z_FULL, stL, 0);
                if (lane == 0) {
                    uint32_t o = st.bits;
                    st.put(o, sM & ((1u << ctM->log) - 1u), 0, ctM->log); o += ctM->log;
                    st.put(o, sO & ((1u << ctO->log) - 1u), 0, ctO->log); o += ctO->log;
                    st.put(o, sL & ((1u << ctL->log) - 1u), 0, ctL->log); o += ctL->log;
                    st.put(o, 1, 0, 1);
                }
                st.bits += ctM->log + ctO->log + ctL->log + 1u;
                st.flush(lane, true);
            }
            seqSecSize += (uint32_t)(st.out - bsStart);
            }
        }
        __syncwarp();
        const uint32_t bodySize = litSecSize + seqSecSize;
        if (!overCap && bodySize < blkSize) {
            if (lane == 0) { const uint32_t h = last | (2u << 1) | (bodySize << 3); out[0] = (uint8_t)h; out[1] = (uint8_t)(h >> 8); out[2] = (uint8_t)(h >> 16); }
            outSize = 3 + bodySize;
        } else {
            if (lane == 0) { const uint32_t h = last | (blkSize << 3); out[0] = (uint8_t)h; out[1] = (uint8_t)(h >> 8); out[2] = (uint8_t)(h >> 16); }
            __syncwarp();
            warp_copy(out + 3, bsrc, blkSize, lane);
            outSize = 3 + blkSize;
        }
        if (lane == 0) slotSize[blk] = outSize;
        __syncwarp();
    }
}

#ifndef B2Z_CUEMU
void launch_zstd_enc_entropy(const uint8_t* src, uint64_t srcSize, const EncGeom& g,
                             const uint64_t* seqs, const uint32_t* nseq, const uint8_t* lits, const uint32_t* nlit,
                             uint8_t* slots, uint32_t* slotSize, uint32_t nBlocks, uint32_t smCount, cudaStream_t st) {
    if (!nBlocks) return;
    uint32_t grid = (nBlocks + B2Z_ENT_WARPS - 1) / B2Z_ENT_WARPS;
    const uint32_t cap = smCount * 16u;
    if (grid > cap) grid = cap;
    zstd_enc_entropy_kernel<<<grid, B2Z_ENT_WARPS * 32, 0, st>>>(src, srcSize, g, seqs, nseq, lits, nlit, slots, slotSize, nBlocks);
}
#endif

}  // namespace b2z
