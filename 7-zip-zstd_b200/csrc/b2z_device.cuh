// b2z_device.cuh -- small device helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "b2z_params.h"

#define B2Z_FULL 0xFFFFFFFFu

namespace b2z {

#ifdef B2Z_CUEMU   // tests/cuemu compiles the kernel sources for the host (logic checks without a GPU): no PTX there
__device__ __forceinline__ uint32_t lane_id() { return cuemu_lane_id(); }
__device__ __forceinline__ uint32_t lanemask_lt() { return (1u << cuemu_lane_id()) - 1u; }
#define B2Z_DYN_SMEM(T, name) T* const name = reinterpret_cast<T*>(cuemu::dyn_smem())
#define B2Z_EXTERN_SMEM(T, name) T* const name = reinterpret_cast<T*>(cuemu::dyn_smem())
__device__ __forceinline__ void bar_sync(uint32_t id, uint32_t nThreads) { cuemu::named_bar(id, nThreads, true); }
__device__ __forceinline__ void bar_arrive(uint32_t id, uint32_t nThreads) { cuemu::named_bar(id, nThreads, false); }
#else
__device__ __forceinline__ uint32_t lane_id() { uint32_t l; asm volatile("mov.u32 %0, %%laneid;" : "=r"(l)); return l; }
__device__ __forceinline__ uint32_t lanemask_lt() { uint32_t m; asm volatile("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }
// the CTA's dynamic shared memory as an array (B2Z_EXTERN_SMEM: exactly `extern __shared__ T name[]`) or as one struct
#define B2Z_EXTERN_SMEM(T, name) extern __shared__ T name[]
#define B2Z_DYN_SMEM(T, name) extern __shared__ __align__(16) unsigned char name##_raw_[]; T* const name = reinterpret_cast<T*>(name##_raw_)
// named barriers (ids 1..15; 0 is __syncthreads): bar_sync waits until nThreads threads have arrived (bar_sync or bar_arrive),
// bar_arrive only signals.  Memory accesses before an arrive are visible after the matching sync (PTX barrier semantics).
__device__ __forceinline__ void bar_sync(uint32_t id, uint32_t nThreads) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nThreads) : "memory"); }
__device__ __forceinline__ void bar_arrive(uint32_t id, uint32_t nThreads) { asm volatile("bar.arrive %0, %1;" :: "r"(id), "r"(nThreads) : "memory"); }
#endif

// 64-bit funnel: bytes [s/8, s/8+8) of the 16-byte little-endian pair (a, b); s in {0,8,..,56}
__device__ __forceinline__ uint64_t funnel64(uint64_t a, uint64_t b, uint32_t s) {
    return (a >> s) | ((b << 1) << (63u - s));
}

// read-only (non-coherent, L1-cacheable) aligned 8-byte load of word `i` of the frame
__device__ __forceinline__ uint64_t ldw(const uint64_t* __restrict__ w, uint32_t i, uint32_t nWords) {
    return i < nWords ? __ldg(w + i) : 0ull;
}

// unaligned 8 bytes at byte offset `o` of a frame whose base is 8-byte aligned; bytes at or
// beyond nWords*8 read as zero (never dereferenced)
__device__ __forceinline__ uint64_t ld64u(const uint64_t* __restrict__ w, uint32_t o, uint32_t nWords) {
    uint32_t i = o >> 3, s = (o & 7u) * 8u;
    uint64_t a = ldw(w, i, nWords), b = s ? ldw(w, i + 1, nWords) : 0ull;
    return funnel64(a, b, s);
}

// common-prefix length of frame[q..] and frame[p..], capped at maxLen (q < p)
__device__ __forceinline__ uint32_t match_len(const uint64_t* __restrict__ w, uint32_t q, uint32_t p,
                                              uint32_t maxLen, uint32_t nWords) {
    uint32_t qi = q >> 3, pi = p >> 3, qs = (q & 7u) * 8u, ps = (p & 7u) * 8u;
    uint64_t qa = ldw(w, qi, nWords), pa = ldw(w, pi, nWords);
    uint32_t len = 0;
    while (len < maxLen) {
        uint64_t qb = ldw(w, qi + 1, nWords), pb = ldw(w, pi + 1, nWords);
        uint64_t x = funnel64(qa, qb, qs) ^ funnel64(pa, pb, ps);
        if (x) { len += (uint32_t)(__ffsll((long long)x) - 1) >> 3; break; }
        len += 8; qa = qb; pa = pb; qi++; pi++;
    }
    return len < maxLen ? len : maxLen;
}

// same, when the first 8 bytes at p are already in a register (`pv`): most candidates differ inside those 8 bytes,
// and then no p-side load is needed at all
__device__ __forceinline__ uint32_t match_len_pv(const uint64_t* __restrict__ w, uint32_t q, uint32_t p, uint64_t pv,
                                                 uint32_t maxLen, uint32_t nWords) {
    const uint32_t qi = q >> 3, qs = (q & 7u) * 8u;
    const uint64_t qa = ldw(w, qi, nWords), qb = ldw(w, qi + 1, nWords);
    const uint64_t x = funnel64(qa, qb, qs) ^ pv;
    uint32_t len;
    if (x) len = (uint32_t)(__ffsll((long long)x) - 1) >> 3;
    else {
        len = 8;
        uint32_t qj = qi + 1, pj = (p >> 3) + 1; const uint32_t ps = (p & 7u) * 8u;
        uint64_t qc = qb, pc = ldw(w, pj, nWords);
        while (len < maxLen) {
            const uint64_t qd = ldw(w, qj + 1, nWords), pd = ldw(w, pj + 1, nWords);
            const uint64_t y = funnel64(qc, qd, qs) ^ funnel64(pc, pd, ps);
            if (y) { len += (uint32_t)(__ffsll((long long)y) - 1) >> 3; break; }
            len += 8; qc = qd; pc = pd; qj++; pj++;
        }
    }
    return len < maxLen ? len : maxLen;
}

// common-prefix length of base[q..] and base[p..] beyond the first `from` bytes (known equal), capped at maxLen; warp-uniform
__device__ __forceinline__ uint32_t warp_extend(const uint8_t* __restrict__ base, uint32_t q, uint32_t p, uint32_t from, uint32_t maxLen, uint32_t lane) {
    for (uint32_t s = from;; s += 32u) {
        const uint32_t k = s + lane;
        const bool eq = k < maxLen && __ldg(base + q + k) == __ldg(base + p + k);
        const uint32_t mism = __ballot_sync(B2Z_FULL, !eq);
        if (mism) return s + (uint32_t)(__ffs((int)mism) - 1);
    }
}

__device__ __forceinline__ uint32_t highbit32(uint32_t v) { return 31u - (uint32_t)__clz((int)v); }

__device__ __forceinline__ uint32_t warp_excl_scan(uint32_t v, uint32_t lane, uint32_t* total) {
    uint32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(B2Z_FULL, x, d); if (lane >= (uint32_t)d) x += y; }
    *total = __shfl_sync(B2Z_FULL, x, 31);
    return x - v;
}

// XXH64 (seed 0) of `len` bytes at an 8-byte aligned address; one thread walks one buffer (four independent
// accumulators give the instruction-level parallelism).  Content checksum of a zstd frame = low 32 bits
// (C/zstd/zstd_compress.c:5344-5400, ../hashes/xxhash.c).
__device__ __forceinline__ uint64_t xxh_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xxh_round(uint64_t acc, uint64_t in) { return xxh_rotl(acc + in * 0xC2B2AE3D27D4EB4Full, 31) * 0x9E3779B185EBCA87ull; }
__device__ __forceinline__ uint64_t xxh_merge(uint64_t h, uint64_t v) { return (h ^ xxh_round(0, v)) * 0x9E3779B185EBCA87ull + 0x85EBCA77C2B2AE63ull; }
__device__ inline uint64_t xxh64_device(const uint8_t* data, uint64_t len) {
    const uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
    const uint64_t* w = reinterpret_cast<const uint64_t*>(data);
    uint64_t i = 0, h;
    if (len >= 32) {
        uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0ull - P1;
        const uint64_t nStripes = len >> 5;
        for (uint64_t k = 0; k < nStripes; k++) { v1 = xxh_round(v1, w[4 * k]); v2 = xxh_round(v2, w[4 * k + 1]); v3 = xxh_round(v3, w[4 * k + 2]); v4 = xxh_round(v4, w[4 * k + 3]); }
        i = nStripes << 5;
        h = xxh_rotl(v1, 1) + xxh_rotl(v2, 7) + xxh_rotl(v3, 12) + xxh_rotl(v4, 18);
        h = xxh_merge(h, v1); h = xxh_merge(h, v2); h = xxh_merge(h, v3); h = xxh_merge(h, v4);
    } else h = P5;
    h += len;
    for (; i + 8 <= len; i += 8) { h ^= xxh_round(0, w[i >> 3]); h = xxh_rotl(h, 27) * P1 + P4; }
    if (i + 4 <= len) { h ^= (uint64_t)(*reinterpret_cast<const uint32_t*>(data + i)) * P1; h = xxh_rotl(h, 23) * P2 + P3; i += 4; }
    for (; i < len; i++) { h ^= data[i] * P5; h = xxh_rotl(h, 11) * P1; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

// same for a buffer at any byte alignment (decoder outputs of frames that follow an odd-sized frame)
__device__ inline uint64_t xxh64_device_unaligned(const uint8_t* data, uint64_t len) {
    const uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
    const uint64_t* w = reinterpret_cast<const uint64_t*>(reinterpret_cast<uintptr_t>(data) & ~(uintptr_t)7);
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(data) & 7u) * 8u;
    auto rd = [&](uint64_t byteOff) -> uint64_t {                     // 8 bytes at data+byteOff (multiple of 8), never reading past data+len
        if (byteOff + 16 <= len) { const uint64_t i = byteOff >> 3; return funnel64(w[i], w[i + 1], sh); }
        uint64_t v = 0; for (int b = 0; b < 8; b++) v |= (uint64_t)data[byteOff + b] << (8 * b); return v;
    };
    uint64_t i = 0, h;
    if (len >= 32) {
        uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0ull - P1;
        const uint64_t nStripes = len >> 5;
        for (uint64_t k = 0; k < nStripes; k++) { v1 = xxh_round(v1, rd(32 * k)); v2 = xxh_round(v2, rd(32 * k + 8)); v3 = xxh_round(v3, rd(32 * k + 16)); v4 = xxh_round(v4, rd(32 * k + 24)); }
        i = nStripes << 5;
        h = xxh_rotl(v1, 1) + xxh_rotl(v2, 7) + xxh_rotl(v3, 12) + xxh_rotl(v4, 18);
        h = xxh_merge(h, v1); h = xxh_merge(h, v2); h = xxh_merge(h, v3); h = xxh_merge(h, v4);
    } else h = P5;
    h += len;
    for (; i + 8 <= len; i += 8) { h ^= xxh_round(0, rd(i)); h = xxh_rotl(h, 27) * P1 + P4; }
    if (i + 4 <= len) { uint32_t v = 0; for (int b = 0; b < 4; b++) v |= (uint32_t)data[i + b] << (8 * b); h ^= (uint64_t)v * P1; h = xxh_rotl(h, 23) * P2 + P3; i += 4; }
    for (; i < len; i++) { h ^= data[i] * P5; h = xxh_rotl(h, 11) * P1; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}


// XXH64 by one warp, for the one big frame the reference's .zst handler writes with a content checksum (ZstdHandler.cpp:262-282).
// The four stripe accumulators are four strictly sequential chains -- lanes 0-3 run one each, dependent 64-bit
// arithmetic per 32 input bytes, which is the floor for this hash on any machine that cannot multiply faster.  What the other lanes
// add is the memory pipeline: the warp loads the next tile (aligned 16-byte words, coalesced, any byte alignment of `data`) into
// registers while the four lanes work on the current one from shared memory.  tileMem: 2 * B2Z_XXH_TILE_BYTES, 16-byte aligned.
#define B2Z_XXH_TILE 4096u
#define B2Z_XXH_TILE_BYTES (B2Z_XXH_TILE + 32u)
#define B2Z_XXH_WS_BYTES (2u * B2Z_XXH_TILE_BYTES + B2Z_XXH_TILE)       /* two raw tiles + the tile's inputs times P2 */
__device__ inline uint64_t xxh64_warp(const uint8_t* data, uint64_t len, uint8_t* tileMem /* B2Z_XXH_WS_BYTES, 16-byte aligned */, uint32_t lane) {
    const uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull, P5 = 0x27D4EB2F165667C5ull;
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(data) & 15u);
    const uint4* __restrict__ aw = reinterpret_cast<const uint4*>(data - sh);            // aligned words; word j holds data bytes [16 j - sh, 16 j - sh + 16)
    const uint64_t nStripes = len >> 5, stripeBytes = nStripes << 5;
    const uint64_t nWordsValid = (sh + len + 15u) >> 4;                                    // words that hold at least one byte of the buffer
    constexpr uint32_t WPT = B2Z_XXH_TILE / 16u + 1u, PER = (WPT + 31u) / 32u;             // words per tile (one more for the shift), per lane
    uint64_t acc = lane == 0 ? P1 + P2 : (lane == 1 ? P2 : (lane == 2 ? 0ull : 0ull - P1));
    const uint64_t nTiles = (stripeBytes + B2Z_XXH_TILE - 1u) / B2Z_XXH_TILE;
    uint64_t* const pre = reinterpret_cast<uint64_t*>(tileMem + 2u * B2Z_XXH_TILE_BYTES);  // pre[m] = (m-th 8-byte input of the tile) * P2
    uint4 r[PER];
    auto fetch = [&](uint64_t t) {
#pragma unroll
        for (uint32_t k = 0; k < PER; k++) {
            const uint32_t j = k * 32u + lane; const uint64_t wj = t * (B2Z_XXH_TILE / 16u) + j;
            r[k] = (j < WPT && wj < nWordsValid) ? aw[wj] : make_uint4(0, 0, 0, 0);
        }
    };
    auto stash = [&](uint32_t buf) {
        uint4* d = reinterpret_cast<uint4*>(tileMem + buf * B2Z_XXH_TILE_BYTES);
#pragma unroll
        for (uint32_t k = 0; k < PER; k++) { const uint32_t j = k * 32u + lane; if (j < WPT) d[j] = r[k]; }
    };
    if (nTiles) { fetch(0); stash(0); }
    __syncwarp();
    for (uint64_t t = 0; t < nTiles; t++) {
        if (t + 1 < nTiles) fetch(t + 1);                                                  // in flight while this tile is hashed
        const uint64_t left = stripeBytes - t * B2Z_XXH_TILE;
        const uint32_t ns = (uint32_t)((left < B2Z_XXH_TILE ? left : B2Z_XXH_TILE) >> 5);
        {   // every lane: the alignment shift and the multiplication by P2, which do not depend on the accumulators
            const uint64_t* w = reinterpret_cast<const uint64_t*>(tileMem + (uint32_t)(t & 1u) * B2Z_XXH_TILE_BYTES);
            const uint32_t bsh = (sh & 7u) * 8u, o0 = (sh & 8u) >> 3;
            for (uint32_t m = lane; m < ns * 4u; m += 32u) pre[m] = funnel64(w[o0 + m], w[o0 + m + 1u], bsh) * P2;
        }
        __syncwarp();
        if (lane < 4u) {                                                                   // the four sequential chains: add, rotate, multiply
            uint32_t k = 0, o = lane;
            for (; k + 8u <= ns; k += 8u, o += 32u) {                                      // eight stripes per pass, their loads first (issue is in order)
                uint64_t in[8];
#pragma unroll
                for (uint32_t j = 0; j < 8u; j++) in[j] = pre[o + 4u * j];
#pragma unroll
                for (uint32_t j = 0; j < 8u; j++) acc = xxh_rotl(acc + in[j], 31) * P1;
            }
            for (; k < ns; k++, o += 4u) acc = xxh_rotl(acc + pre[o], 31) * P1;
        }
        __syncwarp();
        if (t + 1 < nTiles) stash((uint32_t)((t + 1) & 1u));
        __syncwarp();
    }
    const uint64_t v1 = __shfl_sync(B2Z_FULL, acc, 0), v2 = __shfl_sync(B2Z_FULL, acc, 1), v3 = __shfl_sync(B2Z_FULL, acc, 2), v4 = __shfl_sync(B2Z_FULL, acc, 3);
    uint64_t h;
    if (len >= 32) {
        h = xxh_rotl(v1, 1) + xxh_rotl(v2, 7) + xxh_rotl(v3, 12) + xxh_rotl(v4, 18);
        h = xxh_merge(h, v1); h = xxh_merge(h, v2); h = xxh_merge(h, v3); h = xxh_merge(h, v4);
    } else h = P5;
    h += len;
    uint64_t i = stripeBytes;                                                              // < 32 bytes left: every lane repeats them (byte loads)
    for (; i + 8 <= len; i += 8) { uint64_t v = 0; for (int b = 0; b < 8; b++) v |= (uint64_t)data[i + b] << (8 * b); h ^= xxh_round(0, v); h = xxh_rotl(h, 27) * P1 + P4; }
    if (i + 4 <= len) { uint32_t v = 0; for (int b = 0; b < 4; b++) v |= (uint32_t)data[i + b] << (8 * b); h ^= (uint64_t)v * P1; h = xxh_rotl(h, 23) * P2 + P3; i += 4; }
    for (; i < len; i++) { h ^= data[i] * P5; h = xxh_rotl(h, 11) * P1; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

}  // namespace b2z
