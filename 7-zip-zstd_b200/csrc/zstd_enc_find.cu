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
// Per iteration a position takes the turn, compares the candidates it requested one iteration earlier, hashes the next
// iteration's 16 bytes, and requests this iteration's two candidates together with the own bytes two iterations ahead (which an
// L2 prefetch one iteration earlier has brought from DRAM), so a candidate's round trip runs while the group does its next turn.
// Level 3 (<4, 7, 0>, 896 threads): 64 registers, no spills; the GUARD = false loop is 159 SASS instructions per position plus
// the prefetch (cuobjdump -sass).  Stage F per 4 GiB step of the bench: 35.4 -> 31.0 ms on an H100 80GB HBM3 (700 W,
// 1980 MHz); DESIGN 2.2.
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

// 16 bytes at any byte offset as four 32-bit words: the five aligned 32-bit words that hold them (W5, as loaded) and four native
// funnel shifts (shr16; the 64-bit formulation costs eight ALU instructions per 8 bytes).  The two halves are apart so that a
// load can be carried to a later iteration and shifted where it is used.  GUARD: words at or beyond nW4 read as zero (only the
// last frame of a buffer needs it: any other frame is followed by readable bytes, and a length is clipped to the frame anyway).
struct B16 { uint32_t x0, x1, x2, x3; };
struct W5 { uint32_t t0, t1, t2, t3, t4; };
static_assert(B2Z_CAP == 16, "stage F compares four 32-bit words");
// The loads are coherent (ld.global.ca, L1-cached like __ldg): ptxas keeps those in front of a later bar.sync, where it would
// sink non-coherent ones towards their use -- into the turn, or below it.
__device__ __forceinline__ uint32_t ldca(const uint32_t* p) {
#ifndef B2Z_CUEMU
    return __ldca(p);
#else
    return __ldg(p);
#endif
}
template <bool GUARD>
__device__ __forceinline__ W5 ld20(const uint32_t* __restrict__ w4, uint32_t a, uint32_t nW4) {
    W5 r;
    if (!GUARD) { r.t0 = ldca(w4 + a); r.t1 = ldca(w4 + a + 1u); r.t2 = ldca(w4 + a + 2u); r.t3 = ldca(w4 + a + 3u); r.t4 = ldca(w4 + a + 4u); return r; }
    r.t0 = a < nW4 ? ldca(w4 + a) : 0u; r.t1 = a + 1u < nW4 ? ldca(w4 + a + 1u) : 0u; r.t2 = a + 2u < nW4 ? ldca(w4 + a + 2u) : 0u;
    r.t3 = a + 3u < nW4 ? ldca(w4 + a + 3u) : 0u; r.t4 = a + 4u < nW4 ? ldca(w4 + a + 4u) : 0u;
    return r;
}
// The own bytes are the first touch of the input, a DRAM round trip.  Their load shares its scoreboard with the candidates' loads
// (ptxas puts every load of the loop on one), so the wait for the candidates after a turn would also wait for DRAM.  A prefetch
// into L2 one iteration before the load (no register, no scoreboard) turns that load into an L2 hit like the candidates'.
__device__ __forceinline__ void prefetch_l2(const uint32_t* p) {
#ifndef B2Z_CUEMU
    asm volatile("prefetch.global.L2 [%0];" :: "l"(p));
#else
    (void)p;
#endif
}
// (the funnel shift takes its amount mod 32, so byte offset o gives sh = o * 8)
__device__ __forceinline__ B16 shr16(const W5& t, uint32_t sh) {
    B16 r; r.x0 = __funnelshift_r(t.t0, t.t1, sh); r.x1 = __funnelshift_r(t.t1, t.t2, sh); r.x2 = __funnelshift_r(t.t2, t.t3, sh); r.x3 = __funnelshift_r(t.t3, t.t4, sh);
    return r;
}
// common-prefix length (0..15) of two 16-byte strings, or a number above 16 when all 16 bytes agree (__ffs(0) - 1 wraps): the
// caller clips it to at most 16 anyway
__device__ __forceinline__ uint32_t prefix16(const B16& a, const B16& b) {
    const uint32_t d0 = a.x0 ^ b.x0, d1 = a.x1 ^ b.x1, d2 = a.x2 ^ b.x2, d3 = a.x3 ^ b.x3;
    const uint32_t z = d0 ? d0 : (d1 ? d1 : (d2 ? d2 : d3));
    const uint32_t base = d0 ? 0u : (d1 ? 4u : (d2 ? 8u : 12u));
    return base + ((uint32_t)(__ffs((int)z) - 1) >> 3);
}

// MODE 0: both tables (levels 3-4); 1: only the short table (levels 1-2, fast levels); 2: both tables + the lower lanes of a
// position's own step (levels 5-7) -- b2z_params.h: B2Z_FLAG_FIND_FAST / B2Z_FLAG_FIND_STEP
struct FindCtx {
    uint32_t* smem; uint32_t* TL; uint32_t* TS; uint32_t tableWords, HL, HS, tagBits, tagMask, W, tid, grp, tg;
    uint32_t barTurn, barGrp, barNext;                                         // named barrier ids of this thread's group
};

// -DB2Z_F_CLOCKS (off by default; tools/enc_find_profile.py --build-clocks): every warp adds the clock64() cycles it spends in each
// phase to f_clocks[]; b200z_find_clocks() reads and clears them.  Without the switch the ticks compile to nothing.
//   wait: bar.sync of the turn (the previous group still holds it); turn: table reads, group barrier, atomics, hand-over;
//   cand: comparing the previous iteration's candidates (with whatever is left of their round trip); work: hash, the loads, store.
enum { FC_WAIT, FC_TURN, FC_CAND, FC_WORK, FC_N };
#ifdef B2Z_F_CLOCKS
__device__ unsigned long long f_clocks[FC_N + 1];                             // [FC_N] = warps
#define F_TICK(ph) do { const long long now_ = clock64(); fc[ph] += (unsigned long long)(now_ - fcLast); fcLast = now_; } while (0)
#else
#define F_TICK(ph) do { } while (0)
#endif

// One position's candidates, carried from the turn that found them to the next one: where both candidates start, their offsets,
// the lengths they may reach (0 for a candidate that failed its tag or window test), the position's own 16 bytes, and both
// candidates' words as loaded.
struct Pending { B16 own; W5 rL, rS; uint32_t cL, cS, offL, offS, mL, mS; };

// both candidates' words of a pending position (a failed candidate starts at the position itself: no branch between the loads)
template <bool FAST, bool GUARD>
__device__ __forceinline__ void request(Pending& q, const uint32_t* __restrict__ w4, uint32_t nW4) {
    if (!FAST) q.rL = ld20<GUARD>(w4, q.cL >> 2, nW4);
    q.rS = ld20<GUARD>(w4, q.cS >> 2, nW4);
}

// the candidate word of a pending position (B2Z_CAND, 0 = none)
template <bool FAST>
__device__ __forceinline__ uint32_t cand_word(const Pending& q) {
    const uint32_t lL = FAST ? 0u : prefix16(shr16(q.rL, q.cL * 8u), q.own), lS = prefix16(shr16(q.rS, q.cS * 8u), q.own);
    const uint32_t lenL = FAST ? 0u : (lL < q.mL ? lL : q.mL), lenS = lS < q.mS ? lS : q.mS;
    // the longer wins, the nearer of two equally long ones (offsets < 2^24: a frame is at most 2^B2Z_MAX_FRAMELOG bytes); a
    // length below B2Z_DP_MINLEN makes the word 0 whichever side it came from
    const uint32_t kL = (lenL << 24) | (~q.offL & 0xFFFFFFu), kS = (lenS << 24) | (~q.offS & 0xFFFFFFu);
    const uint32_t k = kS > kL ? kS : kL, len = k >> 24;
    return len >= B2Z_DP_MINLEN ? B2Z_CAND(len, ~k & 0xFFFFFFu) : 0u;
}

// the chunks of one frame (n bytes at w4, candidate words to out)
//
// Per position and iteration: take the turn with the hash computed at the end of the previous iteration, compare the previous
// iteration's candidates and store their word, hash the next iteration's 16 bytes (loaded one iteration earlier), then request
// this iteration's candidates and the 16 bytes of the iteration after next.  A candidate's round trip so overlaps the group's
// wait for its next turn instead of following the turn.  The hash comes before the loads because ptxas puts all of them on one
// scoreboard: a wait for the own bytes also waits for every load issued before it.  The last iteration's candidates are
// compared after the loop.  The output pointer and the own bytes' word index advance by a step per iteration; the own bytes'
// shift is fixed per frame (p mod 4 never changes: a step is G * CH positions).
template <int WPG, int G, int MODE, bool GUARD>
__device__ __forceinline__ void find_frame(const FindCtx& c, const uint32_t* __restrict__ w4, uint32_t n, uint32_t* __restrict__ out
#ifdef B2Z_F_CLOCKS
                                           , unsigned long long* fc, long long& fcLast
#endif
                                           ) {
    constexpr uint32_t CH = WPG * 32u, STEPW = G * CH;
    constexpr bool FAST = MODE == 1, STEP = MODE == 2;
    const uint32_t nW4 = (n + 3u) >> 2;
    const uint32_t HL = c.HL, HS = c.HS, tagBits = c.tagBits, W = c.W;
    uint32_t tagMask = c.tagMask;
#ifndef B2Z_CUEMU
    // held in registers for the whole frame: without the opaque moves ptxas recomputes both in the loop (4 + 3 instructions)
    asm("mov.b64 %0, %0;" : "+l"(w4)); asm("mov.b32 %0, %0;" : "+r"(tagMask));
#endif
    constexpr uint64_t PL = B2Z_PRIME8, PS = B2Z_PRIME5 << 24;
    const uint32_t shIL = 32u - HL, shIS = 32u - HS, shTL = 32u - HL - tagBits, shTS = 32u - HS - tagBits;
    const uint32_t nChunks = (n + CH - 1u) / CH, nIter = (nChunks + G - 1u) / G;
    uint32_t p = c.grp * CH + c.tg;
    const uint32_t shOwn = p * 8u;                                        // the own bytes' shift (p mod 4 = tg mod 4 for the whole frame)
    B16 own = shr16(ld20<true>(w4, p >> 2, nW4), shOwn);
    W5 vNext = ld20<true>(w4, (p + STEPW) >> 2, nW4);                     // the next iteration's own bytes ...
    uint32_t aNext = (p >> 2) + 2u * STEPW / 4u;                          // ... and the first word of the ones after them
    uint32_t hl, hs;
    // the index and the tag are the top HL + tagBits bits of the 64-bit product, and HL + tagBits <= 15 + (31 - 17) < 32
    // (launch_zstd_enc_find checks it): only the high word of each product is formed.  (v << 24) * PRIME5 = v * (PRIME5 << 24).
    auto hash = [&]() {
        hl = (uint32_t)(((uint64_t)own.x0 * (uint32_t)PL) >> 32) + own.x0 * (uint32_t)(PL >> 32) + own.x1 * (uint32_t)PL;
        hs = (uint32_t)(((uint64_t)own.x0 * (uint32_t)PS) >> 32) + own.x0 * (uint32_t)(PS >> 32) + own.x1 * (uint32_t)PS;
    };
    hash();
    uint32_t* __restrict__ o = out + p;
    Pending q = {};                                                       // nothing pending before the first iteration (lengths 0)
    for (uint32_t it = 0; it < nIter; it++, p += STEPW, aNext += STEPW / 4u, o += STEPW) {
        // ---- before the turn: table indices and tags of the 16 bytes at p, same-step groups
        const bool hashable = p + 8u <= n;                                 // p >= n for the padding chunks of the last iteration
        const uint32_t iL = hl >> shIL, iS = hs >> shIS;
        const uint32_t tL = (hl >> shTL) & tagMask, tS = (hs >> shTS) & tagMask;
        const uint32_t mineL = ((p + 1u) << tagBits) | tL, mineS = ((p + 1u) << tagBits) | tS;
        // what the turn writes: max with 0 leaves an entry as it is, so a padding position's atomics need no branch
        const uint32_t putL = hashable ? mineL : 0u, putS = hashable ? mineS : 0u;
        uint32_t* const aL = c.TL + iL; uint32_t* const aS = c.TS + iS;
        uint32_t lowL = 0, lowS = 0;
        if (STEP) {                                                        // lanes of this step with my table index, below me
            const uint32_t lane = c.tid & 31u, lt = (1u << lane) - 1u;
            lowL = __match_any_sync(B2Z_FULL, hashable ? iL : (0x80000000u | lane)) & lt;
            lowS = __match_any_sync(B2Z_FULL, hashable ? iS : (0x80000000u | lane)) & lt;
        }
        turn_inputs_ready(c.smem + c.tableWords + c.tid, iL, iS, putL, putS, c.barNext ^ lowL ^ (lowS << 1));
        F_TICK(FC_WORK);
        // ---- the turn: nothing but the table accesses between the two barrier hops
        bar_sync(c.barTurn, 2u * CH);
        F_TICK(FC_WAIT);
        uint32_t eL = 0, eS;
        if (!FAST) eL = *aL;
        eS = *aS;
        if (WPG > 1) bar_sync(c.barGrp, CH); else __syncwarp();
        if (!FAST) atomicMax(aL, putL);                                    // the highest position of the chunk stays
        atomicMax(aS, putS);
        bar_arrive(c.barNext, 2u * CH);
        F_TICK(FC_TURN);
        if (STEP) {                                                        // a lower lane of the step with my index is nearer than the table's entry
            const uint32_t fromL = __shfl_sync(B2Z_FULL, mineL, lowL ? 31 - __clz((int)lowL) : 0);
            const uint32_t fromS = __shfl_sync(B2Z_FULL, mineS, lowS ? 31 - __clz((int)lowS) : 0);
            if (lowL) eL = fromL;
            if (lowS) eS = fromS;
        }
        // ---- after the turn: the previous iteration's word (the branch keeps ptxas from moving the compare into the turn)
        if (p - STEPW < n) {                                               // (p - STEPW wraps around in the first iteration)
            const uint32_t word = cand_word<FAST>(q);
            F_TICK(FC_CAND);
            __stcs(o - STEPW, word);
        }
        const uint32_t offL = p - ((eL >> tagBits) - 1u), offS = p - ((eS >> tagBits) - 1u);
        const bool okL = !FAST && hashable && eL && (eL & tagMask) == tL && offL <= W;
        const bool okS = hashable && eS && (eS & tagMask) == tS && offS <= W && !(okL && offS == offL);   // not the long one's offset
        // at most B2Z_CAP = 16 bytes are compared, never beyond the position's 4 KiB parse segment
        const uint32_t segEnd = ((p | (B2Z_SEG - 1u)) + 1u) < n ? ((p | (B2Z_SEG - 1u)) + 1u) : n;
        const uint32_t maxLen = (segEnd - p) < B2Z_CAP ? (segEnd - p) : B2Z_CAP;
        q.own = own; q.cL = p - (okL ? offL : 0u); q.cS = p - (okS ? offS : 0u); q.offL = offL; q.offS = offS;
        q.mL = okL ? maxLen : 0u; q.mS = okS ? maxLen : 0u;                // (0 for a position that is not hashable)
        // ---- the next iteration's hash, then the loads
        own = shr16(vNext, shOwn);
        hash();
        vNext = GUARD ? ld20<true>(w4, (p + 2u * STEPW) >> 2, nW4) : ld20<false>(w4, aNext, 0u);
        if (!GUARD) prefetch_l2(w4 + aNext + STEPW / 4u);                 // and the ones after those into L2 (see prefetch_l2)
        request<FAST, GUARD>(q, w4, nW4);
    }
    // the last iteration's candidates (p and o are one step past it)
    const uint32_t word = cand_word<FAST>(q);
    if (p - STEPW < n) __stcs(o - STEPW, word);
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
    c.barTurn = B2Z_FIND_BAR_TURN(c.grp); c.barGrp = B2Z_FIND_BAR_GRP(c.grp);
    c.barNext = B2Z_FIND_BAR_TURN(c.grp + 1u == (uint32_t)G ? 0u : c.grp + 1u);
    const uint64_t nFrames = (srcSize + (1ull << g.frameLog) - 1) >> g.frameLog;
    const uint32_t tid = c.tid;
#ifdef B2Z_F_CLOCKS
    unsigned long long fc[FC_N] = {};
    long long fcLast = clock64();
#define B2Z_F_CLOCK_ARGS , fc, fcLast
#else
#define B2Z_F_CLOCK_ARGS
#endif

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
        F_TICK(FC_WORK);
        // a frame followed by at least 4 KiB of the buffer needs no bounds checks on its loads (they reach at most 3 * 896 + 20 bytes
        // past the frame: the own bytes two iterations after a padding chunk; the L2 prefetch of the own bytes one iteration
        // further reaches 4 * 896 bytes)
        if (srcSize - f0 - n >= 4096u) find_frame<WPG, G, MODE, false>(c, w4, n, out B2Z_F_CLOCK_ARGS);
        else find_frame<WPG, G, MODE, true>(c, w4, n, out B2Z_F_CLOCK_ARGS);
    }
#undef B2Z_F_CLOCK_ARGS
    // leave the barriers balanced: the hand-over that closed the last frame is consumed by group 0
    if (c.grp == 0) bar_sync(B2Z_FIND_BAR_TURN(0), 2u * CH);
#ifdef B2Z_F_CLOCKS
    if ((tid & 31u) == 0) { for (int p_ = 0; p_ < FC_N; p_++) atomicAdd(&f_clocks[p_], fc[p_]); atomicAdd(&f_clocks[FC_N], 1ull); }
#endif
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
    // find_frame hashes with the high words of the products only, and packs an offset into 24 bits
    const uint32_t hashLog = g.hashLogL > g.hashLogS ? g.hashLogL : g.hashLogS;
    if (g.frameLog < 17 || g.frameLog > B2Z_MAX_FRAMELOG || hashLog + 31u - g.frameLog > 32u) return cudaErrorInvalidValue;
    switch (g.chunkLog) {
    case 5: return launch_find_t<1, 7>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    case 6: return launch_find_t<2, 7>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    case 7: return launch_find_t<4, 7>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    case 8: return launch_find_t<8, 4>(src, srcSize, g, cand, nCtas, ready, readyShift, errFlag, st);
    }
    return cudaErrorInvalidValue;
}

#ifdef B2Z_F_CLOCKS
// the per-phase cycle sums of every warp since the last call (FC_* order, then the warp count); clears them
extern "C" int b200z_find_clocks(unsigned long long* out) {
    static const unsigned long long zero[FC_N + 1] = {};
    cudaError_t e = cudaMemcpyFromSymbol(out, f_clocks, sizeof(f_clocks));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(f_clocks, zero, sizeof(f_clocks));
    return (int)e;
}
#endif
#endif

}  // namespace b2z
