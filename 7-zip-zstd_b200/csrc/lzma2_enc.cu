// lzma2_enc.cu -- stage R of the block-parallel LZMA2 encoder (7-Zip method 21) for sm_90a.
//
// A frame (2^frameLog input bytes) becomes one dictionary-reset LZMA2 block -- the independent unit the reference's own
// MT coders use (Lzma2Enc.c:241-330 block split; fast-lzma2 slices, lzma2_enc.c:1937-2099).  Stage M (zstd_enc_match.cu,
// shared with the zstd path) -- or, with B2Z_FLAG_LZ2_OPT, stage C + stage P (lzma2_parse.cu: the price-based parse) -- has
// already found the frame's sequences; here one thread per frame codes them as LZMA
// packets with the adaptive binary range coder, which is a strictly serial chain of dependent instructions:
// the parallelism is across frames (thousands per batch), not inside one.
//   model      11-bit probabilities in shared memory (16 KiB, 13 frames/SM) or, when there are more frames than that
//              fills, the 12 KiB literal part in global memory (32 frames/SM)
//   input      bytes the next packet needs (its symbol, the previous byte, the byte at rep0) are loaded before the
//              current packet is coded, so their L2 latency hides under the range coding of the current one
//   chunks     closed at 64 KiB - 64 packed bytes or 2 MiB - 512 covered; a chunk that does not shrink is rewritten as
//              an uncompressed chunk and the next one resets the model (Lzma2Enc.c:183-238)
//
// Replaces (reference, /root/reference/C/): LzmaEnc.c:691-760 (range coder), :795-860 (literals), :934-1010 (lengths),
// :2388-2600 (packets), Lzma2Enc.c:129-238 (chunks), fast-lzma2/range_enc.c, lzma2_enc.c:1937-2099.
// Oracle statement: oracle/lzma2_enc_oracle.c (byte-exact).
#include <cstdlib>
#include "b2z_device.cuh"
#include "b2z_kernels.h"
#include "b2z_lzma2.h"
#include "b2z_params.h"

namespace b2z {

struct RcE {
    uint64_t low; uint32_t range, cacheSize, cache;
    uint8_t* out; uint32_t op;       // out: slot base; op: bytes written so far
};

// Not inlined on purpose: it runs once per ~13 coded bits, and inlining it at the ~25 rce_bit sites (with its byte loop
// unrolled) made the kernel large enough to miss in the instruction cache.
__device__ __noinline__ void rce_shift_low(RcE& e) {
    if ((uint32_t)e.low < 0xFF000000u || (uint32_t)(e.low >> 32) != 0u) {
        const uint32_t carry = (uint32_t)(e.low >> 32);
        uint32_t c = e.cache;
        uint8_t* o = e.out + e.op;
        e.op += e.cacheSize;
#pragma unroll 1
        do { *o++ = (uint8_t)(c + carry); c = 0xFFu; } while (--e.cacheSize != 0u);
        e.cache = ((uint32_t)e.low >> 24) & 0xFFu;
    }
    e.cacheSize++;
    e.low = (e.low & 0x00FFFFFFull) << 8;
}
__device__ __forceinline__ void rce_bit(RcE& e, uint16_t* p, uint32_t bit) {
    const uint32_t v = *p, bound = (e.range >> 11) * v;
    // v += (2048 - v) >> 5  |  v -= v >> 5, as one expression: floor((31 - v) / 32) == -(v >> 5)
    *p = (uint16_t)((int32_t)v + (((bit ? 31 : 2048) - (int32_t)v) >> 5));
    if (!bit) e.range = bound; else { e.low += bound; e.range -= bound; }
    if (e.range < (1u << 24)) { e.range <<= 8; rce_shift_low(e); }     // one step suffices: v >= 31, so range >= 2^13 * 31 before it
}
__device__ __forceinline__ void rce_direct(RcE& e, uint32_t v, uint32_t n) {
    while (n--) {
        e.range >>= 1;
        if ((v >> n) & 1u) e.low += e.range;
        if (e.range < (1u << 24)) { e.range <<= 8; rce_shift_low(e); }
    }
}
__device__ __forceinline__ void rce_tree(RcE& e, uint16_t* p, uint32_t bits, uint32_t v) {
    uint32_t m = 1;
    for (uint32_t i = bits; i--;) { const uint32_t b = (v >> i) & 1u; rce_bit(e, p + m, b); m = (m << 1) | b; }
}
__device__ __forceinline__ void rce_tree_rev(RcE& e, uint16_t* p, uint32_t bits, uint32_t v) {
    uint32_t m = 1;
    for (uint32_t i = 0; i < bits; i++) { const uint32_t b = (v >> i) & 1u; rce_bit(e, p + m, b); m = (m << 1) | b; }
}
__device__ __forceinline__ void rce_len(RcE& e, uint16_t* l, uint32_t len, uint32_t ps) {
    len -= 2u;
    if (len < 8u) { rce_bit(e, l + L_CHOICE, 0); rce_tree(e, l + L_LOW + ps * 8u, 3, len); }
    else if (len < 16u) { rce_bit(e, l + L_CHOICE, 1); rce_bit(e, l + L_CHOICE2, 0); rce_tree(e, l + L_MID + ps * 8u, 3, len - 8u); }
    else { rce_bit(e, l + L_CHOICE, 1); rce_bit(e, l + L_CHOICE2, 1); rce_tree(e, l + L_HIGH, 8, len - 16u); }
}

// L: chains per warp (lanes 0, 32/L, 2*32/L ... each run one chain).  Only L = 1 is launched: L = 2/4/8 measured
// slower -- the chains' control flow diverges at every coded bit, so the hardware
// serialises them and the shared convergent code does not pay for it.
// DYN: lc / lp / pb from the properties byte in g.flags (B2Z_FLAG_LZ2_PROPS); otherwise the defaults, as compile-time constants
template <bool GLIT, int L, bool DYN = false>
// <= 64 registers: they are allocated for all 32 lanes of a chain's warp, so registers -- not shared memory -- bound the
// chains per SM (32 at 64 registers)
__global__ void __launch_bounds__(64, 16)
lzma2_enc_range_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, const uint64_t* __restrict__ seqs,
                       const uint32_t* __restrict__ nseq, uint8_t* __restrict__ slots, uint32_t slotStride,
                       uint32_t* __restrict__ slotSize, uint16_t* __restrict__ litSpill, uint32_t* __restrict__ status, uint32_t nChains) {
    B2Z_EXTERN_SMEM(uint16_t, probsAll);
    constexpr uint32_t LSTEP = 32u / (uint32_t)L;
    if ((threadIdx.x & 31u) % LSTEP) return;                        // one thread per chain; see the header comment
    // chain = (frame, slice): a frame's range coding is split into state-reset slices of sliceBlocks 128 KiB blocks
    const uint32_t slotInCta = (threadIdx.x >> 5) * (uint32_t)L + (threadIdx.x & 31u) / LSTEP;
    const uint32_t chain = blockIdx.x * (blockDim.x >> 5) * (uint32_t)L + slotInCta;
    if (chain >= nChains) return;
    const uint32_t props = DYN ? b2z_lz2_props(g.flags) : B2Z_LZ2_PROPS;
    const uint32_t LC = b2z_lz2_lc(props), LITN = b2z_lz2_litn(props);
    uint16_t* const probs = probsAll + (size_t)slotInCta * (GLIT ? P_LIT : P_LIT + LITN);
    const uint64_t F = 1ull << g.frameLog;
    const uint32_t bpf = (uint32_t)(F >> 17), sliceBlocks = B2Z_LZ2_SLICE_BLOCKS(g.frameLog, g.flags), spf = bpf / sliceBlocks;
    const uint32_t f = chain / spf, sl = chain - f * spf;
    const uint64_t f0 = (uint64_t)f << g.frameLog;
    const uint32_t n = (uint32_t)((srcSize - f0) < F ? (srcSize - f0) : F);
    const uint8_t* __restrict__ base = src + f0;
    const uint32_t nblkFrame = (n + B2Z_BLOCK - 1u) / B2Z_BLOCK;
    const uint32_t b0 = sl * sliceBlocks, b1 = (b0 + sliceBlocks) < nblkFrame ? (b0 + sliceBlocks) : nblkFrame;
    uint16_t* lit = GLIT ? litSpill + (size_t)chain * LITN : probs + P_LIT;
    if (GLIT) asm volatile("" : "+l"(lit));                         // keep the base in registers: ptxas otherwise rebuilds it from the
                                                                    // kernel parameters at every probability access (5 instructions per bit)
    const uint32_t PBM = (1u << b2z_lz2_pb(props)) - 1u, LPM = (1u << b2z_lz2_lp(props)) - 1u;

    RcE e; e.low = 0; e.range = 0; e.cacheSize = 0; e.cache = 0; e.out = slots + (size_t)chain * slotStride; e.op = 0;
    uint32_t state = 0, rep0 = 0, rep1 = 0, rep2 = 0, rep3 = 0;
    uint32_t chunkPos = 0, chunkOut = 0, hdr = 0;
    bool open = false, needDict = sl == 0, needProps = true, needState = true, overflow = false;
    if (b0 >= nblkFrame) { slotSize[chain] = 0; return; }           // slice beyond the end of a short last frame

    auto chunk_close = [&](uint32_t pos) {
        for (int i = 0; i < 5; i++) rce_shift_low(e);
        lzma2_chunk_write(e.out, e.op, chunkOut, hdr, base + chunkPos, pos - chunkPos, props, needDict, needProps, needState);
        open = false;
    };
    auto chunk_step = [&](uint32_t pos) {                           // before every packet
        if (open && (e.op - chunkOut - hdr + e.cacheSize >= B2Z_LZ2_PACK_LIMIT || pos - chunkPos >= B2Z_LZ2_UNPACK_LIMIT)) chunk_close(pos);
        if (!open) {
            if (e.op + 65536u + 96u > slotStride) { overflow = true; return; }
            chunkPos = pos; chunkOut = e.op;
            hdr = (needDict || needProps) ? 6u : 5u;
            if (needDict || needProps || needState) {
                uint32_t* w = reinterpret_cast<uint32_t*>(probs);
                for (uint32_t i = 0; i < (GLIT ? P_LIT : P_LIT + LITN) / 2u; i++) w[i] = 0x04000400u;
                if (GLIT) { uint32_t* gl = reinterpret_cast<uint32_t*>(lit); for (uint32_t i = 0; i < LITN / 2u; i++) gl[i] = 0x04000400u; }
                state = 0; rep0 = rep1 = rep2 = rep3 = 0;
            }
            e.op += hdr;
            e.low = 0; e.range = 0xFFFFFFFFu; e.cache = 0; e.cacheSize = 1;
            open = true;
        }
    };

    // bytes of the packet about to be coded: cur = base[pos], prev = base[pos-1], mb = base[pos-rep0-1] (meaningful when state >= 7)
    uint32_t pos = b0 * B2Z_BLOCK, cur = __ldg(base + pos), prev = pos ? (uint32_t)__ldg(base + pos - 1u) : 0u, mb = 0;

    auto literal = [&]() {
        const uint32_t nxt = (pos + 1u < n) ? (uint32_t)__ldg(base + pos + 1u) : 0u;         // for the next packet
        rce_bit(e, probs + P_ISMATCH + state * 16u + (pos & PBM), 0);
        uint16_t* p = lit + 0x300u * (((pos & LPM) << LC) + (prev >> (8u - LC)));
        uint32_t m = 1, i = 8;
        if (state >= 7u) {                                          // matched literal: context follows the byte at rep0 while it agrees
#pragma unroll 1
            while (i) {
                --i;
                const uint32_t b = (cur >> i) & 1u, mbit = (mb >> i) & 1u;
                rce_bit(e, p + ((1u + mbit) << 8) + m, b);
                m = (m << 1) | b;
                if (mbit != b) break;
            }
        }
        // the tree walk keeps the 64-bit address p + m itself (p + 2m + b = (p + m) + m + b): one wide multiply-add per
        // bit instead of rebuilding the address from the model base
        uint16_t* pm = p + m;
#pragma unroll 1
        while (i) { --i; const uint32_t b = (cur >> i) & 1u; rce_bit(e, pm, b); pm += m + b; m = (m << 1) | b; }
        state = state < 4u ? 0u : (state < 10u ? state - 3u : state - 6u);
        prev = cur; cur = nxt; pos++;
    };
    auto match = [&](uint32_t len, uint32_t dist) {                  // dist = distance - 1
        const uint32_t pN = pos + len;
        const uint32_t nxt = (pN < n) ? (uint32_t)__ldg(base + pN) : 0u, prevN = __ldg(base + pN - 1u), mbN = __ldg(base + pN - dist - 1u);
        const uint32_t ps = pos & PBM;
        rce_bit(e, probs + P_ISMATCH + state * 16u + ps, 1);
        int r = dist == rep0 ? 0 : (dist == rep1 ? 1 : (dist == rep2 ? 2 : (dist == rep3 ? 3 : -1)));
        if (r < 0) {
            rce_bit(e, probs + P_ISREP + state, 0);
            rce_len(e, probs + P_LEN, len, ps);
            state = state < 7u ? 7u : 10u;
            uint32_t slot;
            if (dist < 4u) slot = dist; else { const uint32_t nb = highbit32(dist); slot = (nb << 1) | ((dist >> (nb - 1u)) & 1u); }
            rce_tree(e, probs + P_POSSLOT + (len - 2u < 4u ? len - 2u : 3u) * 64u, 6, slot);
            if (slot >= 4u) {
                const uint32_t fb = (slot >> 1) - 1u, b = (2u | (slot & 1u)) << fb, red = dist - b;
                if (slot < 14u) rce_tree_rev(e, probs + P_SPECPOS + b - slot - 1u, fb, red);
                else { rce_direct(e, red >> 4, fb - 4u); rce_tree_rev(e, probs + P_ALIGN, 4, red & 15u); }
            }
            rep3 = rep2; rep2 = rep1; rep1 = rep0; rep0 = dist;
        } else {
            rce_bit(e, probs + P_ISREP + state, 1);
            if (r == 0) { rce_bit(e, probs + P_ISREPG0 + state, 0); rce_bit(e, probs + P_ISREP0LONG + state * 16u + ps, 1); }
            else {
                rce_bit(e, probs + P_ISREPG0 + state, 1);
                if (r == 1) rce_bit(e, probs + P_ISREPG1 + state, 0);
                else { rce_bit(e, probs + P_ISREPG1 + state, 1); rce_bit(e, probs + P_ISREPG2 + state, (uint32_t)(r - 2)); }
                if (r == 3) rep3 = rep2;
                if (r >= 2) rep2 = rep1;
                rep1 = rep0; rep0 = dist;
            }
            rce_len(e, probs + P_REPLEN, len, ps);
            state = state < 7u ? 8u : 11u;
        }
        cur = nxt; prev = prevN; mb = mbN; pos = pN;
    };

    for (uint32_t b = b0; b < b1 && !overflow; b++) {
        const uint32_t bend = (b + 1u) * B2Z_BLOCK < n ? (b + 1u) * B2Z_BLOCK : n;
        const uint64_t* __restrict__ sq = seqs + ((size_t)f * bpf + b) * B2Z_MAXSEQ;
        const uint32_t ns = nseq[(size_t)f * bpf + b];
        uint32_t z0 = 0, z1 = 0, z2 = 0;                             // zstd repcode history of the block, to undo offBase (Emitter::flush)
        uint64_t sNext = ns ? __ldg(sq) : 0ull;
        for (uint32_t i = 0; i < ns && !overflow; i++) {
            const uint64_t s = sNext;
            if (i + 1u < ns) sNext = __ldg(sq + i + 1u);
            const uint32_t ll = B2Z_SEQ_LL(s), ob = B2Z_SEQ_OFFBASE(s); uint32_t ml = B2Z_SEQ_ML(s), off;
            if (ob > 3u) { off = ob - 3u; z2 = z1; z1 = z0; z0 = off; }
            else {
                const uint32_t idx = ob - 1u + (ll == 0u);
                off = idx == 3u ? z0 - 1u : (idx == 0u ? z0 : (idx == 1u ? z1 : z2));
                if (idx != 0u) { if (idx != 1u) z2 = z1; z1 = z0; z0 = off; }
            }
            for (uint32_t j = 0; j < ll && !overflow; j++) { chunk_step(pos); if (!overflow) literal(); }
            while (ml && !overflow) {
                uint32_t len = ml > B2Z_LZ2_MAXLEN ? B2Z_LZ2_MAXLEN : ml;
                if (ml - len == 1u) len--;
                chunk_step(pos); if (overflow) break;
                match(len, off - 1u); ml -= len;
            }
        }
        while (pos < bend && !overflow) { chunk_step(pos); if (!overflow) literal(); }
    }
    if (open && !overflow) chunk_close(pos);
    if (overflow) atomicOr(status, 1u);
    slotSize[chain] = e.op;
}

// ---------------------------------------------------------------------------------------------------- stage R, 32 chains per warp
// The kernel above spends a warp on one chain: 31 of 32 lanes of every issued instruction are idle, and putting several chains on the
// lanes of one warp (template parameter L) only made it slower because the chains' control flow differs at every coded bit.  What does
// NOT differ is the coding of one binary decision -- load the probability, split the range, adapt, renormalise -- so this kernel separates
// the two: every lane owns a chain and
//   phase A (per lane, divergent but short): turns its next packets into a QUEUE of decisions in shared memory -- (probability index, bit)
//           pairs, 13 + 1 bits each; which probabilities a packet touches and with which bits is a function of the input alone, never of
//           the probabilities -- until the queue holds B2Z_R32_FILL decisions;
//   phase B (lock-step): B2Z_R32_FILL times, all 32 lanes pop a decision and code it.  The probabilities of the steps to come are loaded
//           B2Z_R32_DEPTH steps ahead (a step that adapts one of them marks the slot stale; a stale slot loads again at its turn).
// STATUS: parity-green (bytes of the kernel above) but not the default: it was slower than one chain per warp.
// Why: it executes far fewer instructions per decision, but 16 384 chains are only 512 lock-step warps, a handful per SM, each waiting on
// its own dependent latencies with nothing else to run, while the single-chain kernel is issue-bound with many warps per SM.  Selected with
// B200Z_P_LZMA2_MODEL = 3.
// The models live in global memory, interleaved by lane (probability i of lane l at [i][l]).  Chunk rules are the single-chain kernel's:
// a packet may be queued ahead of its coding only while the chunk cannot reach its packed limit before it (a decision emits at most one
// byte, so `packed + queued < limit` is a proof); near the limit a lane queues one packet at a time and decides with an empty queue, which
// is the sequential rule exactly.  Bytes are those of the kernel above (and of oracle/lzma2_enc_oracle.c).
// Replaces (reference): the per-thread slices of fast-lzma2 (lzma2_enc.c:1937-2099) / range_enc.h:62-108 -- there one slice per CPU thread.
#define B2Z_R32_QCAP   128u      // queue slots per lane (a packet is at most 48 decisions: fill < 32 + 48)
#define B2Z_R32_FILL   32u
#define B2Z_R32_DEPTH  4
#define B2Z_R32_DIRECT 0x1FFFu   // "probability index" of a direct bit (range halves, no model)
#define B2Z_R32_WARPS  2u
#define B2Z_R32_MAX_LCLP 3u     // lc + lp of this kernel: its literal model must fit the 13-bit index (lc + lp = 4 is refused)
static_assert(P_LIT + (0x300u << B2Z_R32_MAX_LCLP) < B2Z_R32_DIRECT, "a queue entry holds a 13-bit probability index");

__device__ __forceinline__ void rce32_shift_low(RcE& e) {
    if ((uint32_t)e.low < 0xFF000000u || (uint32_t)(e.low >> 32) != 0u) {
        const uint32_t carry = (uint32_t)(e.low >> 32);
        uint8_t* o = e.out + e.op;
        o[0] = (uint8_t)(e.cache + carry);
        for (uint32_t k = 1; k < e.cacheSize; k++) o[k] = (uint8_t)(0xFFu + carry);
        e.op += e.cacheSize; e.cacheSize = 0;
        e.cache = ((uint32_t)e.low >> 24) & 0xFFu;
    }
    e.cacheSize++;
    e.low = (e.low & 0x00FFFFFFull) << 8;
}

template <bool DYN = false>     // as the kernel above
__global__ void __launch_bounds__(32 * B2Z_R32_WARPS)
lzma2_enc_range32_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, EncGeom g, const uint64_t* __restrict__ seqs,
                         const uint32_t* __restrict__ nseq, uint8_t* __restrict__ slots, uint32_t slotStride,
                         uint32_t* __restrict__ slotSize, uint16_t* models, uint32_t* __restrict__ status, uint32_t nChains) {
    B2Z_EXTERN_SMEM(uint16_t, queues);
    const uint32_t props = DYN ? b2z_lz2_props(g.flags) : B2Z_LZ2_PROPS;
    const uint32_t LC = b2z_lz2_lc(props), NPROBS = P_LIT + b2z_lz2_litn(props);
    const uint32_t PBM = (1u << b2z_lz2_pb(props)) - 1u, LPM = (1u << b2z_lz2_lp(props)) - 1u;
    const uint32_t lane = threadIdx.x & 31u, wic = threadIdx.x >> 5;
    const uint32_t group = blockIdx.x * (blockDim.x >> 5) + wic, chain = group * 32u + lane;
    uint16_t* const q = queues + (size_t)wic * B2Z_R32_QCAP * 32u + lane;                 // slot s of this lane: q[(s % QCAP) * 32]
    uint16_t* const model = models + (size_t)group * NPROBS * 32u + lane;                 // probability i of this lane: model[i * 32]
    uint32_t head = 0, tail = 0;                                                           // decisions coded / queued so far
    auto put = [&](uint32_t idx, uint32_t bit) { q[(tail & (B2Z_R32_QCAP - 1u)) * 32u] = (uint16_t)((idx << 1) | bit); tail++; };
    auto put_tree = [&](uint32_t base, uint32_t bits, uint32_t v) { uint32_t m = 1; for (uint32_t i = bits; i--;) { const uint32_t b = (v >> i) & 1u; put(base + m, b); m = (m << 1) | b; } };
    auto put_tree_rev = [&](uint32_t base, uint32_t bits, uint32_t v) { uint32_t m = 1; for (uint32_t i = 0; i < bits; i++) { const uint32_t b = (v >> i) & 1u; put(base + m, b); m = (m << 1) | b; } };
    auto put_len = [&](uint32_t l, uint32_t len, uint32_t ps) {
        len -= 2u;
        if (len < 8u) { put(l + L_CHOICE, 0); put_tree(l + L_LOW + ps * 8u, 3, len); }
        else if (len < 16u) { put(l + L_CHOICE, 1); put(l + L_CHOICE2, 0); put_tree(l + L_MID + ps * 8u, 3, len - 8u); }
        else { put(l + L_CHOICE, 1); put(l + L_CHOICE2, 1); put_tree(l + L_HIGH, 8, len - 16u); }
    };

    // the chain (frame, slice) of this lane, as in the kernel above
    const uint64_t F = 1ull << g.frameLog;
    const uint32_t bpf = (uint32_t)(F >> 17), sliceBlocks = B2Z_LZ2_SLICE_BLOCKS(g.frameLog, g.flags), spf = bpf / sliceBlocks;
    const uint32_t f = chain / spf, sl = chain - f * spf;
    const uint64_t f0 = (uint64_t)f << g.frameLog;
    bool done = chain >= nChains;
    const uint32_t n = done ? 0u : (uint32_t)((srcSize - f0) < F ? (srcSize - f0) : F);
    const uint8_t* __restrict__ base = src + (done ? 0ull : f0);
    const uint32_t nblkFrame = (n + B2Z_BLOCK - 1u) / B2Z_BLOCK;
    const uint32_t b0 = sl * sliceBlocks, b1 = (b0 + sliceBlocks) < nblkFrame ? (b0 + sliceBlocks) : nblkFrame;
    if (!done && b0 >= nblkFrame) { slotSize[chain] = 0; done = true; }                   // slice beyond the end of a short last frame

    RcE e; e.low = 0; e.range = 0; e.cacheSize = 0; e.cache = 0; e.out = slots + (size_t)(done ? 0u : chain) * slotStride; e.op = 0;
    uint32_t state = 0, rep0 = 0, rep1 = 0, rep2 = 0, rep3 = 0;
    uint32_t chunkPos = 0, chunkOut = 0, hdr = 0;
    bool open = false, needDict = sl == 0, needProps = true, needState = true, overflow = false, finishing = false;

    auto chunk_close = [&](uint32_t pos) {                                              // (queue empty)
        for (int i = 0; i < 5; i++) rce32_shift_low(e);
        lzma2_chunk_write(e.out, e.op, chunkOut, hdr, base + chunkPos, pos - chunkPos, props, needDict, needProps, needState);
        open = false;
    };
    auto chunk_open = [&](uint32_t pos) {                                               // (queue empty)
        if (e.op + 65536u + 96u > slotStride) { overflow = true; return; }
        chunkPos = pos; chunkOut = e.op;
        hdr = (needDict || needProps) ? 6u : 5u;
        if (needDict || needProps || needState) {
            for (uint32_t i = 0; i < NPROBS; i++) model[i * 32u] = 0x0400u;
            state = 0; rep0 = rep1 = rep2 = rep3 = 0;
        }
        e.op += hdr;
        e.low = 0; e.range = 0xFFFFFFFFu; e.cache = 0; e.cacheSize = 1;
        open = true;
    };

    // the producer's cursor: block b, sequence i of ns, what is left of the current sequence (litLeft literals, then mlLeft match bytes at
    // distance mdist + 1), the zstd repcode history of the block (to undo offBase, Emitter::flush), and the bytes the next packet needs
    uint32_t b = b0, i = 0, ns = 0, bend = 0, litLeft = 0, mlLeft = 0, mdist = 0, z0 = 0, z1 = 0, z2 = 0;
    const uint64_t* __restrict__ sq = seqs;
    uint64_t sNext = 0;
    uint32_t pos = b0 * B2Z_BLOCK, cur = 0, prev = 0, mb = 0;
    auto block_begin = [&]() {
        bend = (b + 1u) * B2Z_BLOCK < n ? (b + 1u) * B2Z_BLOCK : n;
        sq = seqs + ((size_t)f * bpf + b) * B2Z_MAXSEQ;
        ns = nseq[(size_t)f * bpf + b]; i = 0; z0 = z1 = z2 = 0;
        sNext = ns ? __ldg(sq) : 0ull;
    };
    if (!done) { cur = __ldg(base + pos); prev = pos ? (uint32_t)__ldg(base + pos - 1u) : 0u; block_begin(); }

    auto literal = [&]() {
        const uint32_t nxt = (pos + 1u < n) ? (uint32_t)__ldg(base + pos + 1u) : 0u;     // for the next packet
        put(P_ISMATCH + state * 16u + (pos & PBM), 0);
        const uint32_t p = P_LIT + 0x300u * (((pos & LPM) << LC) + (prev >> (8u - LC)));
        uint32_t m = 1; bool matched = state >= 7u;                 // matched literal: the context follows the byte at rep0 while it agrees
#pragma unroll
        for (int k = 7; k >= 0; k--) {                              // one shape for every lane: no early exit
            const uint32_t bt = (cur >> k) & 1u, mbit = (mb >> k) & 1u;
            put(p + (matched ? ((1u + mbit) << 8) : 0u) + m, bt);
            m = (m << 1) | bt;
            matched = matched && mbit == bt;
        }
        state = state < 4u ? 0u : (state < 10u ? state - 3u : state - 6u);
        prev = cur; cur = nxt; pos++;
    };
    auto match = [&](uint32_t len, uint32_t dist) {                  // dist = distance - 1
        const uint32_t pN = pos + len;
        const uint32_t nxt = (pN < n) ? (uint32_t)__ldg(base + pN) : 0u, prevN = __ldg(base + pN - 1u), mbN = __ldg(base + pN - dist - 1u);
        const uint32_t ps = pos & PBM;
        put(P_ISMATCH + state * 16u + ps, 1);
        const int r = dist == rep0 ? 0 : (dist == rep1 ? 1 : (dist == rep2 ? 2 : (dist == rep3 ? 3 : -1)));
        if (r < 0) {
            put(P_ISREP + state, 0);
            put_len(P_LEN, len, ps);
            state = state < 7u ? 7u : 10u;
            uint32_t slot;
            if (dist < 4u) slot = dist; else { const uint32_t nb = highbit32(dist); slot = (nb << 1) | ((dist >> (nb - 1u)) & 1u); }
            put_tree(P_POSSLOT + (len - 2u < 4u ? len - 2u : 3u) * 64u, 6, slot);
            if (slot >= 4u) {
                const uint32_t fb = (slot >> 1) - 1u, bs = (2u | (slot & 1u)) << fb, red = dist - bs;
                if (slot < 14u) put_tree_rev(P_SPECPOS + bs - slot - 1u, fb, red);
                else { for (uint32_t k = fb - 4u; k--;) put(B2Z_R32_DIRECT, ((red >> 4) >> k) & 1u); put_tree_rev(P_ALIGN, 4, red & 15u); }
            }
            rep3 = rep2; rep2 = rep1; rep1 = rep0; rep0 = dist;
        } else {
            put(P_ISREP + state, 1);
            if (r == 0) { put(P_ISREPG0 + state, 0); put(P_ISREP0LONG + state * 16u + ps, 1); }
            else {
                put(P_ISREPG0 + state, 1);
                if (r == 1) put(P_ISREPG1 + state, 0);
                else { put(P_ISREPG1 + state, 1); put(P_ISREPG2 + state, (uint32_t)(r - 2)); }
                if (r == 3) rep3 = rep2;
                if (r >= 2) rep2 = rep1;
                rep1 = rep0; rep0 = dist;
            }
            put_len(P_REPLEN, len, ps);
            state = state < 7u ? 8u : 11u;
        }
        cur = nxt; prev = prevN; mb = mbN; pos = pN;
    };

    for (;;) {
        // ---- phase A: queue packets until B2Z_R32_FILL decisions wait (or the lane has to see its queue drain first).  Every pass of the
        // loop is one packet per lane; the __syncwarp()s are there for the hardware, not for the data: without a convergence point after
        // each section the lanes drift apart and the warp executes them one after the other (the cost of 32
        // serial chains)
        bool blocked = false;
        for (;;) {
            bool go = !done && !finishing && !blocked && tail - head < B2Z_R32_FILL;
            if (!__any_sync(B2Z_FULL, go)) break;
            if (go && !litLeft && !mlLeft) {                                            // next sequence / block tail / next block
                for (;;) {
                    if (i < ns) {
                        const uint64_t s = sNext;
                        if (++i < ns) sNext = __ldg(sq + i);
                        const uint32_t ll = B2Z_SEQ_LL(s), ob = B2Z_SEQ_OFFBASE(s); uint32_t off;
                        if (ob > 3u) { off = ob - 3u; z2 = z1; z1 = z0; z0 = off; }
                        else {
                            const uint32_t idx = ob - 1u + (ll == 0u);
                            off = idx == 3u ? z0 - 1u : (idx == 0u ? z0 : (idx == 1u ? z1 : z2));
                            if (idx != 0u) { if (idx != 1u) z2 = z1; z1 = z0; z0 = off; }
                        }
                        litLeft = ll; mlLeft = B2Z_SEQ_ML(s); mdist = off - 1u;
                        if (litLeft | mlLeft) break;
                        continue;
                    }
                    if (pos < bend) { litLeft = bend - pos; break; }
                    if (++b >= b1) { finishing = true; go = false; break; }
                    block_begin();
                }
            }
            __syncwarp();
            if (go && open) {                                                           // the single-chain kernel's chunk_step, see the header
                const uint32_t packed = e.op - chunkOut - hdr + e.cacheSize, queued = tail - head;
                if (packed + queued >= B2Z_LZ2_PACK_LIMIT || pos - chunkPos >= B2Z_LZ2_UNPACK_LIMIT) {
                    if (queued) { blocked = true; go = false; }
                    else if (packed >= B2Z_LZ2_PACK_LIMIT || pos - chunkPos >= B2Z_LZ2_UNPACK_LIMIT) chunk_close(pos);
                }
            }
            if (go && !open) { chunk_open(pos); if (overflow) { done = true; go = false; atomicOr(status, 1u); slotSize[chain] = e.op; } }
            __syncwarp();
            const bool lit = go && litLeft;
            if (lit) {                                                                  // up to three literals per pass (a match is about as many decisions)
                const uint32_t pk = e.op - chunkOut - hdr + e.cacheSize + (tail - head);
                const bool room = pk + 18u < B2Z_LZ2_PACK_LIMIT && pos + 2u - chunkPos < B2Z_LZ2_UNPACK_LIMIT;   // the chunk rule holds for all three
                const uint32_t c = (room && litLeft >= 3u) ? 3u : (room && litLeft == 2u ? 2u : 1u);
#pragma unroll 1
                for (uint32_t k = 0; k < c; k++) literal();
                litLeft -= c;
            }
            __syncwarp();
            if (go && !lit) {
                uint32_t len = mlLeft > B2Z_LZ2_MAXLEN ? B2Z_LZ2_MAXLEN : mlLeft;
                if (mlLeft - len == 1u) len--;
                match(len, mdist); mlLeft -= len;
            }
            __syncwarp();
        }
        if (finishing && !done && tail == head) { if (open) chunk_close(pos); slotSize[chain] = e.op; done = true; }
        if (__all_sync(B2Z_FULL, done)) break;
        __syncwarp();
        // ---- phase B: every lane codes up to B2Z_R32_FILL of its queued decisions, in lock-step
        const uint32_t myN = done ? 0u : ((tail - head) < B2Z_R32_FILL ? (tail - head) : B2Z_R32_FILL);
        uint32_t maxN = myN;
#pragma unroll
        for (int d = 16; d; d >>= 1) { const uint32_t o = __shfl_xor_sync(B2Z_FULL, maxN, d); maxN = o > maxN ? o : maxN; }
        // slot k of the pipeline holds the decision of step s with s % DEPTH == k and its probability, loaded DEPTH steps ahead.  A step that
        // adapts a probability some slot has already loaded marks that slot stale; a stale slot loads again when its turn comes (rare: the
        // same index within DEPTH decisions).  The stale mark is a flag, not a forwarded value, so that nothing touches a slot's register
        // before its load has had DEPTH steps to arrive (forwarding into it made every step wait for the load it had just issued: 40 % of
        // the kernel's time in the first version)
        uint32_t ent[B2Z_R32_DEPTH], pv[B2Z_R32_DEPTH], stale = 0;
#pragma unroll
        for (int j = 0; j < B2Z_R32_DEPTH; j++) {
            ent[j] = 0xFFFFu; pv[j] = 0;
            if ((uint32_t)j < myN) { ent[j] = q[((head + (uint32_t)j) & (B2Z_R32_QCAP - 1u)) * 32u]; if ((ent[j] >> 1) != B2Z_R32_DIRECT) pv[j] = model[(ent[j] >> 1) * 32u]; }
        }
        for (uint32_t s0 = 0; s0 < maxN; s0 += B2Z_R32_DEPTH) {
#pragma unroll
            for (int k = 0; k < B2Z_R32_DEPTH; k++) {
                const uint32_t s = s0 + (uint32_t)k;
                if (s >= maxN) break;                                                    // (warp-uniform)
                const uint32_t en = ent[k], idx = en >> 1, bit = en & 1u;
                const bool act = s < myN, dir = idx == B2Z_R32_DIRECT;
                uint32_t v = pv[k];
                if (act && ((stale >> k) & 1u)) v = model[idx * 32u];
                stale &= ~(1u << k);
                ent[k] = 0xFFFFu; pv[k] = 0;
                if (s + B2Z_R32_DEPTH < myN) {                                           // issue the loads of step s + DEPTH
                    const uint32_t x = q[((head + s + B2Z_R32_DEPTH) & (B2Z_R32_QCAP - 1u)) * 32u];
                    ent[k] = x;
                    if ((x >> 1) != B2Z_R32_DIRECT) pv[k] = model[(x >> 1) * 32u];
                }
                if (act) {
                    const uint32_t half = e.range >> 1, bound = (e.range >> 11) * v;
                    if (!dir) {
                        model[idx * 32u] = (uint16_t)((int32_t)v + (((bit ? 31 : 2048) - (int32_t)v) >> 5));
#pragma unroll
                        for (int j = 0; j < B2Z_R32_DEPTH; j++) if ((ent[j] >> 1) == idx) stale |= 1u << j;
                    }
                    const uint32_t cut = dir ? half : bound;                              // a direct bit halves the range, no model
                    if (bit) e.low += cut;
                    e.range = dir ? half : (bit ? e.range - bound : bound);
                    if (e.range < (1u << 24)) { e.range <<= 8; rce32_shift_low(e); }
                }
                __syncwarp();                                                            // (convergence, see phase A)
            }
        }
        head += myN;
        __syncwarp();
    }
}

uint32_t lzma2_enc_slices_per_frame(const EncGeom& g) { return (1u << (g.frameLog - 17u)) / B2Z_LZ2_SLICE_BLOCKS(g.frameLog, g.flags); }
// slot of one chain (slice): worst case of its chunk stream while it is being produced
size_t lzma2_enc_slot_stride(const EncGeom& g) {
    const uint32_t sliceBytes = B2Z_LZ2_SLICE_BLOCKS(g.frameLog, g.flags) * B2Z_BLOCK;
    return ((size_t)B2Z_LZ2_FRAME_BOUND(sliceBytes) + 255u) & ~(size_t)255u;
}

// bytes of model memory the lock-step kernel needs for nChains chains (whole groups of 32) with the properties of flags
size_t lzma2_enc_model_bytes(uint32_t nChains, uint32_t flags) { return (size_t)((nChains + 31u) / 32u) * 32u * (P_LIT + b2z_lz2_litn(b2z_lz2_props(flags))) * sizeof(uint16_t); }
// chains per SM whose whole model fits shared memory (one chain per CTA, 1 KiB reserved per CTA)
uint32_t lzma2_enc_smem_chains_per_sm(uint32_t flags) {
    return (uint32_t)((227u * 1024u) / (((size_t)P_LIT + b2z_lz2_litn(b2z_lz2_props(flags))) * sizeof(uint16_t) + 1024));
}

#ifndef B2Z_CUEMU
template <bool DYN>
static void launch_range_kernels(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint64_t* seqs, const uint32_t* nseq,
                                 uint8_t* slots, uint32_t stride, uint32_t* slotSize, uint32_t nChains, uint16_t* litSpill, int mode, bool glit,
                                 size_t smemFull, uint32_t* status, cudaStream_t st, cudaError_t* err) {
    if (mode == 3) {                                                // 32 chains per warp (experimental, see the kernel's header); litSpill holds whole models here (lzma2_enc_model_bytes)
        const uint32_t groups = (nChains + 31u) / 32u;
        lzma2_enc_range32_kernel<DYN><<<(groups + B2Z_R32_WARPS - 1u) / B2Z_R32_WARPS, 32 * B2Z_R32_WARPS, B2Z_R32_WARPS * B2Z_R32_QCAP * 32u * sizeof(uint16_t), st>>>(
            src, srcSize, g, seqs, nseq, slots, stride, slotSize, litSpill, status, nChains);
    } else if (glit) {     // two warps (chains) per CTA: 32 CTAs/SM would otherwise cap residency below the register limit
        lzma2_enc_range_kernel<true, 1, DYN><<<(nChains + 1u) / 2u, 64, 2u * P_LIT * sizeof(uint16_t), st>>>(src, srcSize, g, seqs, nseq, slots, stride, slotSize, litSpill, status, nChains);
    } else {
        *err = cudaFuncSetAttribute(lzma2_enc_range_kernel<false, 1, DYN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemFull);
        if (*err != cudaSuccess) return;
        lzma2_enc_range_kernel<false, 1, DYN><<<nChains, 32, smemFull, st>>>(src, srcSize, g, seqs, nseq, slots, stride, slotSize, nullptr, status, nChains);
    }
}

cudaError_t launch_lzma2_enc_range(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint64_t* seqs, const uint32_t* nseq,
                                   uint8_t* slots, uint32_t* slotSize, uint32_t nFrames, uint16_t* litSpill, uint32_t smCount, int mode,
                                   uint32_t* status, cudaStream_t st) {
    if (!nFrames) return cudaSuccess;
    const uint32_t nChains = nFrames * lzma2_enc_slices_per_frame(g);
    const size_t smemFull = ((size_t)P_LIT + b2z_lz2_litn(b2z_lz2_props(g.flags))) * sizeof(uint16_t);
    const uint32_t slotsResident = lzma2_enc_smem_chains_per_sm(g.flags) * smCount;
    // Literal model in global memory when the chains outnumber the shared-memory slots: more chains resident beat the ~6 extra
    // instructions per literal bit of the global-memory model.
    const bool glit = mode == 2 || (mode == 0 && litSpill && nChains > slotsResident);
    const uint32_t stride = (uint32_t)lzma2_enc_slot_stride(g);
    if (mode == 3 && (!litSpill || b2z_lz2_lc(b2z_lz2_props(g.flags)) + b2z_lz2_lp(b2z_lz2_props(g.flags)) > B2Z_R32_MAX_LCLP)) return cudaErrorInvalidValue;
    cudaError_t e = cudaSuccess;
    // the default properties run the compile-time instantiations; any other lc / lp / pb the run-time ones
    if (g.flags & B2Z_FLAG_LZ2_PROPS) launch_range_kernels<true>(src, srcSize, g, seqs, nseq, slots, stride, slotSize, nChains, litSpill, mode, glit, smemFull, status, st, &e);
    else launch_range_kernels<false>(src, srcSize, g, seqs, nseq, slots, stride, slotSize, nChains, litSpill, mode, glit, smemFull, status, st, &e);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

#endif

// ---------------------------------------------------------------------------------------------------- assembly
__global__ void __launch_bounds__(1024)
lzma2_enc_offsets_kernel(const uint32_t* __restrict__ slotSize, uint32_t nFrames, uint64_t* __restrict__ frameOff, uint64_t* __restrict__ outSize) {
    __shared__ uint64_t warpSum[32];
    __shared__ uint64_t carry;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (uint32_t b0 = 0; b0 < nFrames; b0 += 1024u) {
        const uint32_t i = b0 + tid;
        const uint64_t v = i < nFrames ? slotSize[i] : 0u;
        uint64_t x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(B2Z_FULL, x, d); if (lane >= (uint32_t)d) x += y; }
        if (lane == 31) warpSum[wid] = x;
        __syncthreads();
        if (wid == 0) {
            uint64_t s = warpSum[lane], t = s;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint64_t y = __shfl_up_sync(B2Z_FULL, t, d); if (lane >= (uint32_t)d) t += y; }
            warpSum[lane] = t - s;
        }
        __syncthreads();
        const uint64_t excl = carry + warpSum[wid] + (x - v);
        if (i < nFrames) frameOff[i] = excl;
        __syncthreads();
        if (tid == 1023) carry = excl + v;
        __syncthreads();
    }
    if (tid == 0) { frameOff[nFrames] = carry; *outSize = carry + 1u; }
}

// CTA (x, y): part y of gridDim.y of piece x's slot -> its place in the stream (16-byte stores fed by aligned 4-byte reads)
__global__ void __launch_bounds__(256)
lzma2_enc_gather_kernel(const uint8_t* __restrict__ slots, uint32_t slotStride, const uint32_t* __restrict__ slotSize,
                        const uint64_t* __restrict__ frameOff, uint32_t nFrames, uint8_t* __restrict__ dst) {
    const uint32_t f = blockIdx.x, part = blockIdx.y, tid = threadIdx.x;
    const uint32_t total = slotSize[f];
    const uint32_t per = ((total + gridDim.y - 1u) / gridDim.y + 15u) & ~15u;     // 16-byte aligned split of the slot
    const uint32_t s0 = part * per;
    if (f == nFrames - 1u && part == 0 && tid == 0) dst[frameOff[nFrames]] = 0;     // LZMA2 end marker
    if (s0 >= total) return;
    const uint32_t n = (total - s0) < per ? (total - s0) : per;
    const uint8_t* s = slots + (size_t)f * slotStride + s0;
    uint8_t* d = dst + frameOff[f] + s0;
    const uint32_t head = (uint32_t)((16u - ((uintptr_t)d & 15u)) & 15u);
    const uint32_t h = head < n ? head : n;
    if (tid < h) d[tid] = s[tid];
    const uint32_t body = (n - h) & ~15u;
    const uint32_t sh = (h & 3u) * 8u;
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(s + (h & ~3u));
    uint4* dq = reinterpret_cast<uint4*>(d + h);
    for (uint32_t i = tid; i < body / 16u; i += 256u) {
        const uint32_t* q = sw + i * 4u;
        const uint32_t a0 = q[0], a1 = q[1], a2 = q[2], a3 = q[3], a4 = sh ? q[4] : 0u;
        uint4 v;
        v.x = __funnelshift_r(a0, a1, sh); v.y = __funnelshift_r(a1, a2, sh);
        v.z = __funnelshift_r(a2, a3, sh); v.w = __funnelshift_r(a3, a4, sh);
        dq[i] = v;
    }
    for (uint32_t i = h + body + tid; i < n; i += 256u) d[i] = s[i];
}

#ifndef B2Z_CUEMU
// pieces = chains (frame slices) in stream order
void launch_lzma2_enc_assemble(const uint8_t* slots, const uint32_t* slotSize, uint32_t nPieces, uint32_t slotStride, uint64_t* pieceOff,
                               uint8_t* dst, uint64_t* outSize, cudaStream_t st) {
    if (!nPieces) return;
    lzma2_enc_offsets_kernel<<<1, 1024, 0, st>>>(slotSize, nPieces, pieceOff, outSize);
    lzma2_enc_gather_kernel<<<dim3(nPieces, 4), 256, 0, st>>>(slots, slotStride, slotSize, pieceOff, nPieces, dst);
}
#endif

}  // namespace b2z
