// zstd_enc_find.cu -- stage F of the block-parallel Zstandard encoder (sm_90a): the match finder.
//
// One CTA owns one independent frame (2^frameLog input bytes) and keeps BOTH hash tables of the finder in its shared
// memory (long: 2^hashLogL entries indexed by the 8-byte hash, short: 2^hashLogS entries indexed by the 5-byte hash;
// 128 + 64 KiB by default): no table access ever leaves the SM.  An entry is (position + 1) << tagBits | tag, so a
// candidate is only compared with the input when the tag agrees, and atomicMax on an entry keeps the highest position.
//
// The frame is walked in CHUNKS of CH = 32 * WPG positions, thread = position.  The CTA is G groups of WPG warps; chunk c
// belongs to group c mod G.  A chunk's table accesses form a TURN: read both entries (table state before the chunk),
// group barrier, atomicMax both entries, hand the turn to the next group (bar.arrive on its named barrier; the next
// group's bar.sync waits for it).  Everything else -- loading the bytes, hashing, comparing the candidates with the input,
// packing the result -- happens outside the turn, so while one group holds the turn the other G-1 groups hash or compare.  The serial chain of a frame is therefore two shared-memory accesses and two barrier
// hops per CH positions; the result is the pure function of the frame's bytes that
// oracle/zstd_enc_oracle.c:b2zo_zstd_candidates states position by position.
//
// Output: one candidate word per position (B2Z_CAND: offset << 7 | length, 0 = none), consumed by stage G
// (zstd_enc_dp.cu).  Replaces the finder half of zstd_double_fast.c:103-330 (ZSTD_compressBlock_doubleFast_noDict_generic:
// hashLong / hashSmall look-ups and inserts, ZSTD_count), the table upkeep of zstd_compress.c:4591 and the job slicing of
// zstdmt_compress.c:1184-1246 (a frame is a job).
#include "b2z_device.cuh"
#include "b2z_kernels.h"

namespace b2z {

#define B2Z_FIND_BAR_TURN(g) (1u + (g))        // named barrier ids: turn hand-over into group g ...
#define B2Z_FIND_BAR_GRP(g)  (8u + (g))        // ... and the read -> write barrier inside group g

// Keeps everything a turn consumes computed BEFORE its barrier.  ptxas is free to sink arithmetic (and the wait for the bytes'
// global load) below bar.sync, i.e. into the frame's serial chain; a shared-memory store of a word that depends on all of the
// turn's inputs cannot cross the barrier, so the inputs are in registers when the turn begins.
__device__ __forceinline__ void turn_inputs_ready(uint32_t* slot, uint32_t iL, uint32_t iS, uint32_t mineL, uint32_t mineS, uint32_t flags) {
#ifndef B2Z_CUEMU
    const uint32_t mix = iL ^ (iS << 8) ^ mineL ^ (mineS >> 3) ^ flags;
    asm volatile("st.volatile.shared.u32 [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(slot)), "r"(mix) : "memory");
#else
    (void)slot; (void)iL; (void)iS; (void)mineL; (void)mineS; (void)flags;
#endif
}

// 16 bytes at any byte offset as four 32-bit words: five aligned 32-bit loads and four native funnel shifts (the 64-bit formulation
// costs eight ALU instructions per 8 bytes; the ALU pipe is this kernel's bound).  GUARD: words at or beyond nW4 read as zero (only
// the last frame of a buffer needs it: any other frame is followed by readable bytes, and a length is clipped to the frame anyway).
struct B16 { uint32_t x0, x1, x2, x3; };
static_assert(B2Z_CAP == 16, "stage F compares four 32-bit words");
template <bool GUARD>
__device__ __forceinline__ B16 ld16(const uint32_t* __restrict__ w4, uint32_t o, uint32_t nW4) {
    const uint32_t a = o >> 2, sh = (o & 3u) * 8u;
    uint32_t t0, t1, t2, t3, t4;
    if (GUARD) {
        t0 = a < nW4 ? __ldg(w4 + a) : 0u; t1 = a + 1u < nW4 ? __ldg(w4 + a + 1u) : 0u; t2 = a + 2u < nW4 ? __ldg(w4 + a + 2u) : 0u;
        t3 = a + 3u < nW4 ? __ldg(w4 + a + 3u) : 0u; t4 = a + 4u < nW4 ? __ldg(w4 + a + 4u) : 0u;
    } else { t0 = __ldg(w4 + a); t1 = __ldg(w4 + a + 1u); t2 = __ldg(w4 + a + 2u); t3 = __ldg(w4 + a + 3u); t4 = __ldg(w4 + a + 4u); }
    B16 r; r.x0 = __funnelshift_r(t0, t1, sh); r.x1 = __funnelshift_r(t1, t2, sh); r.x2 = __funnelshift_r(t2, t3, sh); r.x3 = __funnelshift_r(t3, t4, sh);
    return r;
}
// common-prefix length (0..16) of two 16-byte strings
__device__ __forceinline__ uint32_t prefix16(const B16& a, const B16& b) {
    const uint32_t d0 = a.x0 ^ b.x0, d1 = a.x1 ^ b.x1, d2 = a.x2 ^ b.x2, d3 = a.x3 ^ b.x3;
    const uint32_t z = d0 ? d0 : (d1 ? d1 : (d2 ? d2 : d3));
    const uint32_t base = d0 ? 0u : (d1 ? 4u : (d2 ? 8u : 12u));
    return z ? base + ((uint32_t)(__ffs((int)z) - 1) >> 3) : 16u;
}

// MODE 0: both tables (levels 3-4); 1: only the short table (levels 1-2, fast levels); 2: both tables + the lower lanes of a
// position's own step (levels 5-7) -- b2z_params.h: B2Z_FLAG_FIND_FAST / B2Z_FLAG_FIND_STEP
struct FindCtx {
    uint32_t* smem; uint32_t* TL; uint32_t* TS; uint32_t tableWords, HL, HS, tagBits, tagMask, W, tid, grp, tg, nextGrp;
};

// the chunks of one frame (n bytes at w4, candidate words to out)
template <int WPG, int G, int MODE, bool GUARD>
__device__ __forceinline__ void find_frame(const FindCtx& c, const uint32_t* __restrict__ w4, uint32_t n, uint32_t* __restrict__ out) {
    constexpr uint32_t CH = WPG * 32u;
    constexpr bool FAST = MODE == 1, STEP = MODE == 2;
    const uint32_t nW4 = (n + 3u) >> 2;
    const uint32_t HL = c.HL, HS = c.HS, tagBits = c.tagBits, tagMask = c.tagMask;
    const uint32_t nChunks = (n + CH - 1u) / CH, nIter = (nChunks + G - 1u) / G;
    B16 vNext = ld16<true>(w4, c.grp * CH + c.tg, nW4);
    for (uint32_t it = 0; it < nIter; it++) {
        const uint32_t p = (it * G + c.grp) * CH + c.tg;
        // ---- before the turn: the 16 bytes at p (loaded one iteration ahead), hashes, same-step groups
        const B16 own = vNext;
        const uint64_t v = (uint64_t)own.x0 | ((uint64_t)own.x1 << 32);
        const bool hashable = p + 8u <= n;                                 // p >= n for the padding chunks of the last iteration
        const uint64_t hl = v * B2Z_PRIME8, hs = (v << 24) * B2Z_PRIME5;
        const uint32_t iL = (uint32_t)(hl >> (64u - HL)), iS = (uint32_t)(hs >> (64u - HS));
        const uint32_t tL = (uint32_t)(hl >> (64u - HL - tagBits)) & tagMask, tS = (uint32_t)(hs >> (64u - HS - tagBits)) & tagMask;
        const uint32_t mineL = ((p + 1u) << tagBits) | tL, mineS = ((p + 1u) << tagBits) | tS;
        uint32_t* const aL = c.TL + iL; uint32_t* const aS = c.TS + iS;
        uint32_t lowL = 0, lowS = 0;
        if (STEP) {                                                        // lanes of this step with my table index, below me
            const uint32_t lane = c.tid & 31u, lt = (1u << lane) - 1u;
            lowL = __match_any_sync(B2Z_FULL, hashable ? iL : (0x80000000u | lane)) & lt;
            lowS = __match_any_sync(B2Z_FULL, hashable ? iS : (0x80000000u | lane)) & lt;
        }
        turn_inputs_ready(c.smem + c.tableWords + c.tid, iL, iS, mineL, mineS, (uint32_t)hashable ^ lowL ^ (lowS << 1));
        // ---- the turn: nothing but the table accesses between the two barrier hops
        bar_sync(B2Z_FIND_BAR_TURN(c.grp), 2u * CH);
        uint32_t eL = 0, eS = 0;
        if (hashable) { if (!FAST) eL = *aL; eS = *aS; }
        if (WPG > 1) bar_sync(B2Z_FIND_BAR_GRP(c.grp), CH); else __syncwarp();
        if (hashable) { if (!FAST) atomicMax(aL, mineL); atomicMax(aS, mineS); }     // the highest position of the chunk stays
        bar_arrive(B2Z_FIND_BAR_TURN(c.nextGrp), 2u * CH);
        if (STEP) {                                                        // a lower lane of the step with my index is nearer than the table's entry
            const uint32_t fromL = __shfl_sync(B2Z_FULL, mineL, lowL ? 31 - __clz((int)lowL) : 0);
            const uint32_t fromS = __shfl_sync(B2Z_FULL, mineS, lowS ? 31 - __clz((int)lowS) : 0);
            if (lowL) eL = fromL;
            if (lowS) eS = fromS;
        }
        // ---- after the turn: the next iteration's bytes are requested before this one's candidates are compared
        vNext = ld16<GUARD>(w4, p + G * CH, nW4);
        uint32_t word = 0;
        if (hashable) {
            // at most B2Z_CAP = 16 bytes are compared, never beyond the position's 4 KiB parse segment
            const uint32_t segEnd = ((p | (B2Z_SEG - 1u)) + 1u) < n ? ((p | (B2Z_SEG - 1u)) + 1u) : n;
            const uint32_t maxLen = (segEnd - p) < B2Z_CAP ? (segEnd - p) : B2Z_CAP;
            uint32_t lenL = 0, offL = 0, lenS = 0, offS = 0;
            if (eL && (eL & tagMask) == tL) { const uint32_t q = (eL >> tagBits) - 1u; if (p - q <= c.W) { offL = p - q; const uint32_t l = prefix16(ld16<GUARD>(w4, q, nW4), own); lenL = l < maxLen ? l : maxLen; } }
            if (eS && (eS & tagMask) == tS) { const uint32_t q = (eS >> tagBits) - 1u; if (p - q <= c.W && p - q != offL) { offS = p - q; const uint32_t l = prefix16(ld16<GUARD>(w4, q, nW4), own); lenS = l < maxLen ? l : maxLen; } }
            uint32_t len = lenL, off = offL;
            if (lenS > lenL || (lenS == lenL && lenS && offS < offL)) { len = lenS; off = offS; }
            if (len >= B2Z_DP_MINLEN) word = B2Z_CAND(len, off);
        }
        if (p < n) __stcs(out + p, word);                                  // streaming: the words are next read by another kernel
    }
}

template <int WPG, int G, int MODE>
__global__ void __launch_bounds__(WPG * G * 32, 1)
zstd_enc_find_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, uint32_t* __restrict__ cand,
                     const volatile uint32_t* ready, uint32_t readyShift, uint32_t* __restrict__ errFlag) {
    B2Z_EXTERN_SMEM(uint32_t, smem);
    constexpr uint32_t CH = WPG * 32u, NT = CH * G;
    static_assert(G >= 2 && G <= 7, "named barriers 1..7 and 8..14");
    FindCtx c;
    c.tid = threadIdx.x; c.grp = c.tid / CH; c.tg = c.tid % CH;
    c.HL = g.hashLogL; c.HS = g.hashLogS;
    c.smem = smem;
    c.TL = smem;                                                              // (MODE 1 keeps no long table: the short one starts the buffer)
    c.TS = smem + (MODE == 1 ? 0u : (1u << c.HL));
    c.tableWords = (MODE == 1 ? 0u : (1u << c.HL)) + (1u << c.HS);
    c.tagBits = 32u - (g.frameLog + 1u); c.tagMask = (1u << c.tagBits) - 1u;
    c.W = g.windowLog >= 32 ? 0xFFFFFFFFu : (1u << g.windowLog);
    c.nextGrp = c.grp + 1u == (uint32_t)G ? 0u : c.grp + 1u;
    const uint64_t nFrames = (srcSize + (1ull << g.frameLog) - 1) >> g.frameLog;
    const uint32_t tid = c.tid;

    // the first turn of the kernel belongs to group 0 and nobody hands it over: the last group arrives once up front.
    // Afterwards every frame runs a multiple of G chunks, so the hand-over that closes a frame opens the next one.
    if (c.grp == (uint32_t)G - 1u) bar_arrive(B2Z_FIND_BAR_TURN(0), 2u * CH);

    for (uint64_t f = blockIdx.x; f < nFrames; f += gridDim.x) {
        const uint64_t f0 = f << g.frameLog;
        const uint32_t n = enc_frame_bytes(g, srcSize, f);
        const uint32_t* __restrict__ w4 = reinterpret_cast<const uint32_t*>(src + f0);
        uint32_t* __restrict__ out = cand + f0;
        // host-pointer path: the input is still being uploaded chunk by chunk; a frame starts once the flag of the chunk
        // that holds its last byte is set (a stream-ordered copy after the chunk).  A flag that never comes is an error
        // the caller sees (B200Z_E_CUDA), never a frame of whatever the buffer held.
        if (ready && n) {
            if (tid == 0) {
                uint32_t spins = 0;
                while (ready[(f0 + n - 1u) >> readyShift] == 0u) { if (++spins > (1u << 22)) { atomicExch(errFlag, 1u); break; } __nanosleep(1000); }
            }
        }
        __syncthreads();                                                       // flag seen; previous frame's table accesses done
        for (uint32_t i = tid; i < c.tableWords / 4u; i += NT) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        // a frame followed by at least 4 KiB of the buffer needs no bounds checks on its loads (they reach at most 2 * 896 + 20 bytes
        // past the frame: the prefetch of a padding chunk)
        if (srcSize - f0 - n >= 4096u) find_frame<WPG, G, MODE, false>(c, w4, n, out);
        else find_frame<WPG, G, MODE, true>(c, w4, n, out);
    }
    // leave the barriers balanced: the hand-over that closed the last frame is consumed by group 0
    if (c.grp == 0) bar_sync(B2Z_FIND_BAR_TURN(0), 2u * CH);
}

#ifndef B2Z_CUEMU
size_t zstd_enc_find_smem_bytes(const EncGeom& g) {          // tables + one scratch word per thread
    return (((g.flags & B2Z_FLAG_FIND_FAST) ? 0 : ((size_t)1 << g.hashLogL)) + ((size_t)1 << g.hashLogS) + 1024u) * 4u;
}

template <int WPG, int G, int MODE>
static cudaError_t launch_find_m(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t* cand, uint32_t nCtas,
                                 const uint32_t* ready, uint32_t readyShift, uint32_t* errFlag, cudaStream_t st) {
    const size_t smem = zstd_enc_find_smem_bytes(g);
    cudaError_t e = cudaFuncSetAttribute(zstd_enc_find_kernel<WPG, G, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   // per device: set on every launch
    if (e != cudaSuccess) return e;
    zstd_enc_find_kernel<WPG, G, MODE><<<nCtas, WPG * G * 32, smem, st>>>(src, srcSize, g, cand, ready, readyShift, errFlag);
    return cudaGetLastError();
}
template <int WPG, int G>
static cudaError_t launch_find_t(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t* cand, uint32_t nCtas,
                                 const uint32_t* ready, uint32_t readyShift, uint32_t* errFlag, cudaStream_t st) {
    if (g.flags & B2Z_FLAG_FIND_FAST) return launch_find_m<WPG, G, 1>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    if (g.flags & B2Z_FLAG_FIND_STEP) return launch_find_m<WPG, G, 2>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    return launch_find_m<WPG, G, 0>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
}

cudaError_t launch_zstd_enc_find(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t* cand, uint32_t nCtas,
                                 const uint32_t* ready, uint32_t readyShift, uint32_t* errFlag, cudaStream_t st) {
    if (srcSize == 0) return cudaSuccess;
    switch (g.chunkLog) {
    case 5: return launch_find_t<1, 7>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    case 6: return launch_find_t<2, 7>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    case 7: return launch_find_t<4, 7>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    case 8: return launch_find_t<8, 4>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    }
    return cudaErrorInvalidValue;
}
#endif

}  // namespace b2z
