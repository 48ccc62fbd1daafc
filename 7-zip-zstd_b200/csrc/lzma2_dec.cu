// lzma2_dec.cu -- block-parallel LZMA2 decoder (7-Zip method 21) for sm_90a.
//
// Pre-pass  lzma2_walk_kernel    one thread hops over the chunk headers (<= 64 KiB of payload per hop) and cuts
//                                the stream at dictionary resets -> Lz2Block[] with output offsets.
// Decode    lzma2_decode_kernel  one warp per block.  The adaptive binary range decoder is a strictly serial
//                                bit chain, so lane 0 owns it (range/code/state/reps in registers, the 11-bit
//                                probability model of the block in shared memory: 3.6 KiB + 1.5 KiB << (lc+lp));
//                                the whole warp serves the three bulk jobs lane 0 hands out:
//                                  MATCH  copy len bytes from distance rep0+1 (periodic extension when they overlap)
//                                  RAW    copy an uncompressed chunk
//                                  RESET  re-initialise the probability model
//                                The output buffer itself is the dictionary (a block never looks behind its own reset).
//
// Replaces (reference, /root/reference/C/): Lzma2DecMt.c:237-414 (block discovery), Lzma2Dec.c:97-330 (chunk FSM),
// LzmaDec.c:229-600 (LZMA_DECODE_REAL), LzmaDec.c:560-640 (match copy / WriteRem).  Oracle: oracle/lzma2_dec_oracle.c.
#include "b2z_device.cuh"
#include "b2z_dec.h"
#include "b2z_lzma2.h"

namespace b2z {

// ---------------------------------------------------------------------------------------------------- pre-pass
struct Lz2EmitDev {
    Lz2Block* blocks; uint32_t cap;
    __host__ __device__ void operator()(uint32_t i, uint64_t s0, uint64_t s1, uint64_t d0, uint64_t dn) const {
        if (i < cap) { Lz2Block b; b.srcOff = s0; b.srcEnd = s1; b.dstOff = d0; b.dstSize = dn; blocks[i] = b; }
    }
};

__global__ void lzma2_walk_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, Lz2Block* blocks, uint32_t cap, Lz2Counts* counts) {
    if (threadIdx.x || blockIdx.x) return;
    Lz2Counts c;
    lzma2_walk(src, srcSize, c, Lz2EmitDev{blocks, cap});
    *counts = c;
}

#ifndef B2Z_CUEMU
void launch_lzma2_walk(const uint8_t* src, uint64_t srcSize, Lz2Block* blocks, uint32_t cap, Lz2Counts* counts, cudaStream_t st) {
    lzma2_walk_kernel<<<1, 32, 0, st>>>(src, srcSize, blocks, cap, counts);
}
#endif

enum : uint32_t { OP_END = 0, OP_MATCH = 1, OP_RAW = 2, OP_RESET = 3, OP_ERROR = 4 };

struct Rc {
    uint32_t range, code, next;       // next: the byte at base[ip], loaded ahead of its use
    uint32_t ip, end;                 // offsets from base (a chunk packs <= 64 KiB)
    const uint8_t* base;
};

__device__ __forceinline__ void rc_norm(Rc& r) {
    if (r.range < (1u << 24)) {
        r.range <<= 8; r.code = (r.code << 8) | r.next;
        ++r.ip;
        // the byte at `end` exists (next chunk header or the end marker); beyond it only a corrupt chunk reads
        r.next = (r.ip <= r.end) ? (uint32_t)__ldg(r.base + r.ip) : 0u;
    }
}
__device__ __forceinline__ uint32_t rc_bit(Rc& r, uint16_t* p) {
    rc_norm(r);
    const uint32_t v = *p;
    const uint32_t bound = (r.range >> 11) * v;
    const uint32_t bit = r.code >= bound ? 1u : 0u;
    // v += (2048 - v) >> 5  |  v -= v >> 5 as one expression: floor((31 - v) / 32) == -(v >> 5)
    *p = (uint16_t)((int32_t)v + (((bit ? 31 : 2048) - (int32_t)v) >> 5));
    if (bit) { r.range -= bound; r.code -= bound; } else r.range = bound;
    return bit;
}
__device__ __forceinline__ uint32_t rc_direct(Rc& r, uint32_t n) {
    uint32_t x = 0;
    while (n--) {
        rc_norm(r);
        r.range >>= 1; r.code -= r.range;
        const uint32_t t = 0u - (r.code >> 31); r.code += r.range & t;
        x = (x << 1) + (t + 1u);
    }
    return x;
}
__device__ __forceinline__ uint32_t rc_tree(Rc& r, uint16_t* p, uint32_t bits) {
    uint32_t m = 1;
    for (uint32_t i = 0; i < bits; i++) m = (m << 1) | rc_bit(r, p + m);
    return m - (1u << bits);
}
__device__ __forceinline__ uint32_t rc_tree_rev(Rc& r, uint16_t* p, uint32_t bits) {
    uint32_t m = 1, x = 0;
    for (uint32_t i = 0; i < bits; i++) { const uint32_t b = rc_bit(r, p + m); m = (m << 1) | b; x |= b << i; }
    return x;
}
__device__ __forceinline__ uint32_t rc_len(Rc& r, uint16_t* l, uint32_t ps) {
    if (!rc_bit(r, l + L_CHOICE)) return 2u + rc_tree(r, l + L_LOW + ps * 8u, 3);
    if (!rc_bit(r, l + L_CHOICE2)) return 10u + rc_tree(r, l + L_MID + ps * 8u, 3);
    return 18u + rc_tree(r, l + L_HIGH, 8);
}

// ---------------------------------------------------------------------------------------------------- decode
// GLIT: the literal model (0x300 << (lc+lp) probabilities, 12 KiB at lc=3) lives in global memory (L1/L2-cached) instead
// of shared memory, which lifts residency from 13 to 32 warps per SM -- used when there are more blocks than smem slots.
template <bool GLIT>
__global__ void __launch_bounds__(32)
lzma2_decode_kernel(const uint8_t* __restrict__ src, const Lz2Block* __restrict__ blocks, uint8_t* __restrict__ dst,
                    uint32_t dictSize, Lz2Counts* counts, uint16_t* __restrict__ litSpill, uint32_t litStride) {
    B2Z_EXTERN_SMEM(uint16_t, probs);
    const uint32_t lane = threadIdx.x;
    uint16_t* const lit = GLIT ? litSpill + (size_t)blockIdx.x * litStride : probs + P_LIT;
    const Lz2Block b = blocks[blockIdx.x];
    uint8_t* const out = dst + b.dstOff;
    const uint8_t* const blkEnd = src + b.srcEnd;
    const uint32_t blkSize = (uint32_t)b.dstSize;

    // lane-0 decoder state
    Rc rc; rc.range = 0; rc.code = 0; rc.next = 0; rc.ip = 0; rc.end = 0; rc.base = src + b.srcOff;
    uint32_t mbNext = 0; bool mbValid = false;     // the byte a matched literal needs right after a match, loaded during the copy
    const uint8_t* hp = src + b.srcOff;            // next chunk header
    uint32_t state = 0, rep0 = 0, rep1 = 0, rep2 = 0, rep3 = 0, lc = 0, lp = 0, pb = 0, prev = 0;
    uint32_t pos = 0, chunkEnd = 0, needInit = 0xE0, litCount = 0;
    bool inChunk = false, pendingInit = false;
    const uint8_t* rawSrc = nullptr;

    for (;;) {
        uint32_t op = OP_END, a = 0, d = 0;
        if (lane == 0) {
            for (;;) {
                if (pos == chunkEnd && !pendingInit) {
                    if (inChunk) {                                  // a finished LZMA chunk: exact size, code == 0 (LzmaDec.c:1020)
                        rc_norm(rc);
                        inChunk = false;
                        if (rc.ip != rc.end || rc.code != 0) { op = OP_ERROR; break; }
                    }
                    if (hp >= blkEnd) { op = (pos == blkSize) ? OP_END : OP_ERROR; break; }
                    // an end marker cannot occur before blkEnd (the walk stops there)
                    const Lz2Chunk ch = lzma2_chunk(hp, (uint64_t)(blkEnd - hp), needInit);
                    if (ch.status || ch.kind == LZ2_CHUNK_END || ch.unpack > blkSize - pos) { op = OP_ERROR; break; }
                    const uint8_t* const payload = hp + ch.hdr;
                    hp = payload + ch.pack;
                    if (ch.kind == LZ2_CHUNK_STORED) { rawSrc = payload; op = OP_RAW; a = ch.unpack; d = pos; pos += ch.unpack; chunkEnd = pos; break; }
                    if (ch.mode >= 2) { lc = ch.lc; lp = ch.lp; pb = ch.pb; litCount = 0x300u << (lc + lp); }
                    if (ch.pack < 5) { op = OP_ERROR; break; }
                    rc.base = payload; rc.ip = 0; rc.end = ch.pack;
                    chunkEnd = pos + ch.unpack; pendingInit = true;
                    if (ch.mode >= 1) { state = 0; rep0 = rep1 = rep2 = rep3 = 0; op = OP_RESET; a = P_LIT + litCount; break; }
                }
                if (pendingInit) {                                  // range decoder start: 0x00 + 4 bytes big-endian (LzmaDec.c:987-998)
                    pendingInit = false; inChunk = true;
                    if (rc.base[0] != 0) { op = OP_ERROR; break; }
                    rc.code = ((uint32_t)rc.base[1] << 24) | ((uint32_t)rc.base[2] << 16) | ((uint32_t)rc.base[3] << 8) | rc.base[4];
                    rc.range = 0xFFFFFFFFu; rc.ip = 5; rc.next = (uint32_t)__ldg(rc.base + 5);
                    mbValid = false;
                }
                // ---- one packet
                const uint32_t ps = pos & ((1u << pb) - 1u);
                if (!rc_bit(rc, probs + P_ISMATCH + state * 16u + ps)) {
                    uint16_t* p = lit + 0x300u * (((pos & ((1u << lp) - 1u)) << lc) + (prev >> (8u - lc)));
                    uint32_t sym = 1;
                    if (state >= 7) {
                        uint32_t mb = mbValid ? mbNext : (uint32_t)out[pos - rep0 - 1u];
                        do {
                            const uint32_t mbit = (mb >> 7) & 1u; mb <<= 1;
                            const uint32_t bit = rc_bit(rc, p + ((1u + mbit) << 8) + sym);
                            sym = (sym << 1) | bit;
                            if (mbit != bit) break;
                        } while (sym < 0x100u);
                    }
                    // the tree walk carries the address p + sym itself: p + 2 sym + b = (p + sym) + sym + b
                    for (uint16_t* pm = p + sym; sym < 0x100u;) { const uint32_t b_ = rc_bit(rc, pm); pm += sym + b_; sym = (sym << 1) | b_; }
                    prev = sym & 0xFFu; mbValid = false;
                    out[pos++] = (uint8_t)prev;
                    state = state < 4 ? 0 : (state < 10 ? state - 3 : state - 6);
                    continue;
                }
                uint32_t len;
                if (!rc_bit(rc, probs + P_ISREP + state)) {
                    rep3 = rep2; rep2 = rep1; rep1 = rep0;
                    len = rc_len(rc, probs + P_LEN, ps);
                    state = state < 7 ? 7 : 10;
                    const uint32_t ls = len - 2u < 4u ? len - 2u : 3u;
                    const uint32_t slot = rc_tree(rc, probs + P_POSSLOT + ls * 64u, 6);
                    if (slot < 4) rep0 = slot;
                    else {
                        const uint32_t nb = (slot >> 1) - 1u;
                        rep0 = (2u | (slot & 1u)) << nb;
                        if (slot < 14) rep0 += rc_tree_rev(rc, probs + P_SPECPOS + rep0 - slot - 1u, nb);
                        else { rep0 += rc_direct(rc, nb - 4u) << 4; rep0 += rc_tree_rev(rc, probs + P_ALIGN, 4); }
                    }
                } else {
                    if (pos == 0) { op = OP_ERROR; break; }
                    if (!rc_bit(rc, probs + P_ISREPG0 + state)) {
                        if (!rc_bit(rc, probs + P_ISREP0LONG + state * 16u + ps)) {
                            state = state < 7 ? 9 : 11;
                            if (rep0 >= pos || rep0 >= dictSize) { op = OP_ERROR; break; }
                            prev = mbValid ? mbNext : (uint32_t)out[pos - rep0 - 1u];     // same byte a matched literal would use
                            mbValid = false;
                            out[pos++] = (uint8_t)prev;
                            continue;
                        }
                    } else {
                        uint32_t dd;
                        if (!rc_bit(rc, probs + P_ISREPG1 + state)) dd = rep1;
                        else { if (!rc_bit(rc, probs + P_ISREPG2 + state)) dd = rep2; else { dd = rep3; rep3 = rep2; } rep2 = rep1; }
                        rep1 = rep0; rep0 = dd;
                    }
                    len = rc_len(rc, probs + P_REPLEN, ps);
                    state = state < 7 ? 8 : 11;
                }
                if (rep0 >= pos || rep0 >= dictSize || len > chunkEnd - pos) { op = OP_ERROR; break; }
                op = OP_MATCH; a = len; d = pos;
                pos += len;
                break;
            }
        }
        op = __shfl_sync(B2Z_FULL, op, 0);
        if (op == OP_END) break;
        if (op == OP_ERROR) { if (lane == 0) atomicOr(&counts->status, B2Z_DERR_CORRUPT); break; }
        a = __shfl_sync(B2Z_FULL, a, 0); d = __shfl_sync(B2Z_FULL, d, 0);
        if (op == OP_MATCH) {
            const uint32_t dist = __shfl_sync(B2Z_FULL, rep0, 0) + 1u;
            __syncwarp();                                           // lane 0's literal stores are visible to the copying lanes
            uint8_t* o = out + d; const uint8_t* s = o - dist;
            uint32_t last = 0;
            if (lane == 0) { mbNext = s[a < dist ? a : a % dist]; mbValid = true; }      // out[pos - rep0 - 1] for the packet after this match
            if (dist >= a) { for (uint32_t i = lane; i < a; i += 32u) { last = s[i]; o[i] = (uint8_t)last; } }
            else { for (uint32_t i = lane; i < a; i += 32u) { last = s[i % dist]; o[i] = (uint8_t)last; } }
            __syncwarp();
            prev = __shfl_sync(B2Z_FULL, last, (a - 1u) & 31u);
        } else if (op == OP_RAW) {
            const uint8_t* s = (const uint8_t*)__shfl_sync(B2Z_FULL, (unsigned long long)rawSrc, 0);
            uint8_t* o = out + d;
            for (uint32_t i = lane; i < a; i += 32u) o[i] = __ldg(s + i);
            __syncwarp();
            prev = __ldg(s + a - 1u);
        } else {                                                    // OP_RESET: a = number of probabilities in use
            uint32_t* w = reinterpret_cast<uint32_t*>(probs);
            if (GLIT) {
                for (uint32_t i = lane; i < P_LIT / 2u; i += 32u) w[i] = 0x04000400u;
                uint32_t* g = reinterpret_cast<uint32_t*>(lit);
                for (uint32_t i = lane; i < (a - P_LIT) / 2u; i += 32u) g[i] = 0x04000400u;
            } else {
                for (uint32_t i = lane; i < (a + 1u) / 2u; i += 32u) w[i] = 0x04000400u;
            }
            __syncwarp();
        }
    }
}

size_t lzma2_lit_spill_bytes(uint32_t nBlocks, uint32_t maxLcLp) { return (size_t)nBlocks * ((size_t)0x300 << maxLcLp) * sizeof(uint16_t); }

#ifndef B2Z_CUEMU
// mode: 0 = choose by block count, 1 = literal model in shared memory, 2 = literal model in global memory (litSpill required)
cudaError_t launch_lzma2_decode(const uint8_t* src, const Lz2Block* blocks, uint32_t nBlocks, uint32_t maxLcLp, uint32_t dictSize,
                                uint8_t* dst, Lz2Counts* counts, uint16_t* litSpill, uint32_t smCount, int mode, cudaStream_t st) {
    if (!nBlocks) return cudaSuccess;
    const uint32_t litCount = 0x300u << maxLcLp;
    const size_t smemFull = ((size_t)P_LIT + litCount) * sizeof(uint16_t);
    const uint32_t slots = (uint32_t)((227u * 1024u) / (smemFull + 1024)) * smCount;       // resident warps with the model in smem
    const bool glit = mode == 2 || (mode == 0 && litSpill && nBlocks > slots);
    if (glit) {
        lzma2_decode_kernel<true><<<nBlocks, 32, P_LIT * sizeof(uint16_t), st>>>(src, blocks, dst, dictSize, counts, litSpill, litCount);
    } else {
        cudaError_t e = cudaFuncSetAttribute(lzma2_decode_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemFull);
        if (e != cudaSuccess) return e;
        lzma2_decode_kernel<false><<<nBlocks, 32, smemFull, st>>>(src, blocks, dst, dictSize, counts, nullptr, 0);
    }
    return cudaGetLastError();
}
#endif

}  // namespace b2z
