// b2z_filter.cu -- the pre/post filters that sit in front of the main coder in a 7z folder or an xz filter chain, on the GPU
// (SURVEY.md 8(f) item 3): Delta, the stateless branch converters ARM64, ARM, PPC, SPARC, and x86, ARM Thumb, RISC-V.  In place on a
// device buffer.
//
//   bra_kernel     one thread per 4-byte instruction: the rule of b2z_filter_ops.h applied to the word with its address -- the
//                  converters C/Bra.c:75-252 run as sequential loops are pure per-instruction functions.  16 B per thread, coalesced.
//   delta          encode: out[i] = in[i] - in[i - d], every byte independent (delta_enc_kernel reads the ORIGINAL neighbour: the
//                  launch goes through a scratch copy).  Decode: per residue class i mod d a running sum, done in three steps:
//                  column sums of tiles of `rows` x d bytes, an exclusive scan of those sums across tiles, then each tile adds its
//                  carry while it accumulates (C/Delta.c:20-169 is the sequential statement).
//   x86_kernel     the x86 BCJ scan carries a 3-bit history from byte to byte (C/Bra86.c:50-170), but the history dies after three
//                  non-opcode bytes: the buffer falls into clusters of E8 / E9 bytes that convert independently; threads find the
//                  cluster starts in their 32-byte spans and run the sequential rule per cluster (b2z_filter_ops.h).
//   armt_kernel    ARM Thumb BL pairs cannot overlap, so they too convert independently: one thread per halfword position.
//   riscv_*        the RISC-V scan steps 2..8 bytes at a time and where it lands depends on every step before: per 64-byte chunk a map
//                  of the four possible entry offsets to the next chunk's, composed by a scan across the buffer, then every chunk
//                  converts from its true entry (below, before riscv_map_kernel).
//   not here       BCJ2 (four output streams + a range coder), IA64 -- B200Z_E_UNSUPPORTED.
// Oracle statements: oracle/filter_oracle.c, tests/riscv_oracle.c (RISC-V); both are checked against the reference's functions
// (oracle/_ref/libref_xz.so).
#include "b2z_device.cuh"
#include "b2z_filter_ops.h"
#ifndef B2Z_CUEMU
#include "b2z_ctx.h"
#endif

namespace b2z {

__global__ void __launch_bounds__(256)
bra_kernel(uint32_t* __restrict__ words, uint64_t nWords, uint32_t kind, int enc, uint32_t startOffset, uint32_t unitLog) {
    // unitLog != 0: the buffer is a run of independent units of 2^unitLog bytes (xz Blocks): addresses restart in each
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t unitMask = unitLog ? ((1ull << unitLog) - 1ull) : ~0ull;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nWords; i += stride) {
        const uint32_t raw = words[i], ia = startOffset + (uint32_t)((i << 2) & unitMask);
        uint32_t out;
        if (kind == B200Z_F_ARM64) out = b2z_conv_arm64(raw, ia, enc);
        else if (kind == B200Z_F_ARM) out = b2z_conv_arm(raw, ia, enc);
        else if (kind == B200Z_F_PPC) out = b2z_bswap32(b2z_conv_ppc(b2z_bswap32(raw), ia, enc));
        else out = b2z_bswap32(b2z_conv_sparc(b2z_bswap32(raw), ia, enc));
        if (out != raw) words[i] = out;
    }
}

// ARM Thumb: one thread per halfword position p (2-byte aligned, p + 4 <= n rounded down to even): a BL pair at p converts on its own
// (b2z_filter_ops.h).  Reads the ORIGINAL halfwords (`in`), writes to `out` (a copy of `in`): a neighbour's result is never an input.
__global__ void __launch_bounds__(256)
armt_kernel(const uint16_t* __restrict__ in, uint16_t* __restrict__ out, uint64_t nHalf, int enc, uint32_t startOffset, uint32_t unitLog) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t unitHalf = unitLog ? (1ull << (unitLog - 1u)) : ~0ull;          // halfwords per independent unit
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i + 1 < nHalf; i += stride) {
        const uint64_t inUnit = unitLog ? (i & (unitHalf - 1ull)) : i;
        if (unitLog && inUnit + 1 >= unitHalf) continue;                           // a pair never straddles two units
        uint32_t h0 = in[i], h1 = in[i + 1];
        if (!b2z_armt_is_bl(h0, h1)) continue;
        b2z_conv_armt(&h0, &h1, startOffset + (uint32_t)(inUnit << 1), enc);
        out[i] = (uint16_t)h0; out[i + 1] = (uint16_t)h1;
    }
}

// x86 BCJ: thread t looks at positions [t * 32, t * 32 + 32) of the ORIGINAL bytes (`in`) for cluster starts -- an opcode byte (E8 / E9
// with 5 bytes left) with no opcode byte in the three positions before it -- and converts each cluster it finds from its start, with
// the sequential rule, until four positions pass without an opcode byte.  Clusters touch disjoint bytes; every decision reads `in`
// (a conversion's operand is never looked at again by the scan), results go to `out`, which starts as a copy of `in`.
__global__ void __launch_bounds__(128)
x86_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, uint64_t nAll, uint32_t pc, int enc, uint32_t unitLog) {
    // unitLog != 0: independent units of 2^unitLog bytes (xz Blocks; a multiple of the 32-byte span): the scan, its history and the
    // addresses restart in each, and a unit's last four bytes are never converted
    const uint64_t tAll = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 32u;
    if (tAll >= nAll) return;
    const uint64_t u0 = unitLog ? (tAll >> unitLog) << unitLog : 0ull;              // this span's unit = [u0, u0 + n)
    const uint64_t n = unitLog ? ((nAll - u0) < (1ull << unitLog) ? (nAll - u0) : (1ull << unitLog)) : nAll;
    in += u0; out += u0;
    const uint64_t t0 = tAll - u0;
    if (n < 5u || t0 > n - 5u) return;
    const uint64_t last = n - 5u;                                   // last position that can hold a convertible opcode
    uint32_t back = 0;                                              // opcode flags of the three positions before c (bit 0 = c - 1)
    for (uint32_t k = 1; k <= 3u; k++) if (t0 >= k && b2z_x86_is_opcode(in[t0 - k])) back |= 1u << (k - 1u);
    for (uint64_t c = t0; c < t0 + 32u && c <= last; c++) {
        const bool op = b2z_x86_is_opcode(in[c]);
        if (op && back == 0u) {                                     // ---- a cluster starts here
            uint32_t hist = 0; uint64_t i = c, rawLast = c;
            while (i <= last) {
                if (i - rawLast > 3u) break;                        // three non-opcode bytes passed: whatever follows is another cluster
                const uint32_t b = in[i];
                if (!b2z_x86_is_opcode(b)) { hist >>= 1; i++; continue; }
                rawLast = i;
                const uint32_t operand = (uint32_t)in[i + 1] | ((uint32_t)in[i + 2] << 8) | ((uint32_t)in[i + 3] << 16) | ((uint32_t)in[i + 4] << 24);
                uint32_t v;
                if (!b2z_x86_convert(hist, operand, pc + (uint32_t)i + 5u, enc, &v)) { hist = (hist >> 1) | 4u; i++; continue; }
                out[i + 1] = (uint8_t)v; out[i + 2] = (uint8_t)(v >> 8); out[i + 3] = (uint8_t)(v >> 16); out[i + 4] = (uint8_t)(v >> 24);
                for (uint32_t k = 1; k <= 4u; k++) if (i + k <= last && b2z_x86_is_opcode(in[i + k])) rawLast = i + k;   // skipped, but they keep the cluster going
                hist = 0; i += 5;
            }
        }
        back = ((back << 1) | (op ? 1u : 0u)) & 7u;
    }
}

__global__ void __launch_bounds__(256)
delta_enc_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, uint64_t n, uint32_t dist, uint32_t unitLog) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t unitMask = unitLog ? ((1ull << unitLog) - 1ull) : ~0ull;     // unitLog != 0: the history restarts every 2^unitLog bytes
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = (uint8_t)(in[i] - ((i & unitMask) >= dist ? in[i - dist] : 0));
}

// tile t = bytes [t * rows * dist, (t + 1) * rows * dist): thread c < dist owns column c (one residue class inside the tile)
__global__ void __launch_bounds__(256)
delta_colsum_kernel(const uint8_t* __restrict__ data, uint64_t n, uint32_t dist, uint32_t rows, uint8_t* __restrict__ sums /* [tiles][dist] */) {
    const uint32_t c = threadIdx.x;
    if (c >= dist) return;
    const uint64_t t0 = (uint64_t)blockIdx.x * rows * dist;
    uint32_t s = 0;
    for (uint32_t r = 0; r < rows; r++) { const uint64_t i = t0 + (uint64_t)r * dist + c; if (i >= n) break; s += data[i]; }
    sums[(uint64_t)blockIdx.x * dist + c] = (uint8_t)s;
}
__global__ void __launch_bounds__(256)
delta_scan_kernel(uint8_t* __restrict__ sums, uint32_t tiles, uint32_t dist) {           // exclusive scan down each column, one CTA
    const uint32_t c = threadIdx.x;
    if (c >= dist) return;
    uint32_t run = 0;
    for (uint32_t t = 0; t < tiles; t++) { const uint32_t v = sums[(uint64_t)t * dist + c]; sums[(uint64_t)t * dist + c] = (uint8_t)run; run += v; }
}
__global__ void __launch_bounds__(256)
delta_dec_kernel(uint8_t* __restrict__ data, uint64_t n, uint32_t dist, uint32_t rows, const uint8_t* __restrict__ carry) {
    const uint32_t c = threadIdx.x;
    if (c >= dist) return;
    const uint64_t t0 = (uint64_t)blockIdx.x * rows * dist;
    uint32_t s = carry[(uint64_t)blockIdx.x * dist + c];
    for (uint32_t r = 0; r < rows; r++) { const uint64_t i = t0 + (uint64_t)r * dist + c; if (i >= n) break; s += data[i]; data[i] = (uint8_t)s; }
}

// ---- RISC-V (b2z_filter_ops.h): a scan with a data-dependent step of 2..8 bytes.  Which positions it visits is a pure function of
// the input, and a step never exceeds 8, so the scan enters a chunk of B2Z_RV_CHUNK bytes at one of four offsets {0, 2, 4, 6}:
//   riscv_map_kernel    one thread per chunk walks the rule from each of the four entries and records where each walk enters the next
//                       chunk -- a map {0..3} -> {0..3} in one byte (2 bits per entry); the CTA's maps are composed into one per CTA
//   riscv_scan_kernel   one CTA: the CTAs' entries, by an exclusive scan of map composition (associative, identity 0xE4)
//   riscv_conv_kernel   each CTA scans its chunks' maps from its entry; each thread then walks its chunk from its own entry, converting
// The walks read the staged original (`in`, padded to whole CTA spans + 8 bytes); conversions go to `out`.  A conversion near the end
// of a chunk writes up to 6 bytes of the next chunk, all before that chunk's entry: every byte has one writer.  unitLog != 0: the
// scan, the addresses and the limit restart in every unit (the last chunk of a unit maps every entry to 0).
#define B2Z_RV_CHUNK 64u
#define B2Z_RV_THREADS 256u
#define B2Z_RV_ROW 72u                                              // chunk + 8 look-ahead bytes; 18 words: 2-way bank conflicts at most
#define B2Z_RV_SPAN (B2Z_RV_CHUNK * B2Z_RV_THREADS)
#define B2Z_RV_ID 0xE4u                                             // the identity map [0, 1, 2, 3]

// f after g: (f o g)(i) = f(g(i))
__device__ __forceinline__ uint32_t rv_compose(uint32_t f, uint32_t g) {
    uint32_t r = 0;
#pragma unroll
    for (uint32_t i = 0; i < 4u; i++) r |= ((f >> (2u * ((g >> (2u * i)) & 3u))) & 3u) << (2u * i);
    return r;
}
// exclusive scan of the CTA's maps in thread order: -> maps[0 .. t) composed; *total = all of them (smem: one word per warp)
__device__ __forceinline__ uint32_t rv_cta_scan(uint32_t m, uint32_t* warpTot, uint32_t* total) {
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    uint32_t inc = m;
#pragma unroll
    for (uint32_t d = 1; d < 32u; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, inc, d);
        if (lane >= d) inc = rv_compose(inc, o);
    }
    uint32_t exc = __shfl_up_sync(0xFFFFFFFFu, inc, 1);
    if (lane == 0) exc = B2Z_RV_ID;
    if (lane == 31u) warpTot[w] = inc;
    __syncthreads();
    uint32_t pre = B2Z_RV_ID;
    for (uint32_t k = 0; k < w; k++) pre = rv_compose(warpTot[k], pre);
    uint32_t all = B2Z_RV_ID;
    for (uint32_t k = 0; k < blockDim.x / 32u; k++) all = rv_compose(warpTot[k], all);
    *total = all;
    return rv_compose(exc, pre);
}
// the CTA's span of `in` -> rows of B2Z_RV_ROW bytes: chunk t's bytes, then the first 8 of chunk t + 1
__device__ __forceinline__ void rv_stage(const uint8_t* __restrict__ in, uint8_t* rows) {
    const uint8_t* src = in + (uint64_t)blockIdx.x * B2Z_RV_SPAN;
    for (uint32_t i = threadIdx.x; i < B2Z_RV_SPAN / 16u; i += blockDim.x) {
        const uint4 v = *(const uint4*)(src + (uint64_t)i * 16u);
        uint2* d = (uint2*)(rows + (i >> 2) * B2Z_RV_ROW + (i & 3u) * 16u);
        d[0] = make_uint2(v.x, v.y); d[1] = make_uint2(v.z, v.w);
    }
    *(uint2*)(rows + threadIdx.x * B2Z_RV_ROW + B2Z_RV_CHUNK) = *(const uint2*)(src + (uint64_t)(threadIdx.x + 1u) * B2Z_RV_CHUNK);
    __syncthreads();
}
__device__ __forceinline__ uint32_t rv_half(const uint8_t* row, uint32_t p) { return *(const uint16_t*)(row + p); }
__device__ __forceinline__ uint32_t rv_word(const uint8_t* row, uint32_t p) { return rv_half(row, p) | (rv_half(row, p + 2u) << 16); }
__device__ __forceinline__ uint32_t rv_step(const uint8_t* row, uint32_t p) {           // b2z_riscv_scan, reading w1 only for candidates
    const uint32_t op = rv_half(row, p) & 0x7Fu;
    if (op != 0x6Fu && op != 0x17u) return 2u;
    return b2z_riscv_scan(rv_word(row, p), rv_word(row, p + 4u));
}
// chunk geometry: [base, base + 64) lies in the unit starting at u0; positions p (chunk-relative) with p < *end are scanned; *last:
// the chunk is the last one of its unit
__device__ __forceinline__ void rv_chunk(uint64_t base, uint64_t n, uint32_t unitLog, uint64_t* u0, uint32_t* end, bool* last) {
    const uint64_t s = unitLog ? (base >> unitLog) << unitLog : 0ull;
    const uint64_t len = unitLog ? ((n - s) < (1ull << unitLog) ? (n - s) : (1ull << unitLog)) : n;
    const uint64_t lim = s + (len & ~1ull);                        // the last position scanned is lim - 8
    *u0 = s;
    *end = lim < base + 8u ? 0u : (lim - 8u - base >= B2Z_RV_CHUNK ? B2Z_RV_CHUNK : (uint32_t)(lim - 8u - base) + 1u);
    *last = base + B2Z_RV_CHUNK >= s + len;
}

__global__ void __launch_bounds__(B2Z_RV_THREADS)
riscv_map_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t unitLog, uint8_t* __restrict__ maps, uint8_t* __restrict__ ctaMaps) {
    __shared__ __align__(16) uint8_t rows[B2Z_RV_THREADS * B2Z_RV_ROW];
    __shared__ uint32_t warpTot[B2Z_RV_THREADS / 32u];
    rv_stage(in, rows);
    const uint64_t chunk = (uint64_t)blockIdx.x * B2Z_RV_THREADS + threadIdx.x, base = chunk * B2Z_RV_CHUNK;
    uint32_t m = B2Z_RV_ID;
    if (base < n) {
        uint64_t u0; uint32_t end; bool last;
        rv_chunk(base, n, unitLog, &u0, &end, &last);
        const uint8_t* row = rows + threadIdx.x * B2Z_RV_ROW;
        // walk from each entry; a walk that reaches a position an earlier walk visited shares that walk's exit
        uint32_t seen[4], exitOf[4];
        m = 0;
#pragma unroll
        for (uint32_t e = 0; e < 4u; e++) {
            uint32_t before = 0;
#pragma unroll
            for (uint32_t k = 0; k < e; k++) before |= seen[k];
            uint32_t p = 2u * e, mine = 0;
            while (p < end && !((before >> (p >> 1)) & 1u)) { mine |= 1u << (p >> 1); p += rv_step(row, p) & ~1u; }
            uint32_t x = 0;                                         // a walk stopped by the limit: no later position is scanned
            if (p >= B2Z_RV_CHUNK) x = (p - B2Z_RV_CHUNK) >> 1;
            else if (p < end) {
#pragma unroll
                for (uint32_t k = 0; k < e; k++) if ((seen[k] >> (p >> 1)) & 1u) x = exitOf[k];
            }
            seen[e] = mine; exitOf[e] = x;
            m |= x << (2u * e);
        }
        if (last) m = 0;                                            // the next chunk starts a unit: entry 0 whatever comes in
        maps[chunk] = (uint8_t)m;
    }
    uint32_t total;
    rv_cta_scan(m, warpTot, &total);
    if (threadIdx.x == 0) ctaMaps[blockIdx.x] = (uint8_t)total;
}

// one CTA of 1024 threads: ctaMaps[b] (CTA b's composed map) -> entry[b] (the offset at which the scan enters CTA b's span)
__global__ void __launch_bounds__(1024)
riscv_scan_kernel(const uint8_t* __restrict__ ctaMaps, uint8_t* __restrict__ entry, uint32_t nCta) {
    __shared__ uint32_t warpTot[32];
    const uint32_t per = (nCta + blockDim.x - 1u) / blockDim.x, lo = threadIdx.x * per, hi = lo + per < nCta ? lo + per : nCta;
    uint32_t m = B2Z_RV_ID;
    for (uint32_t b = lo; b < hi; b++) m = rv_compose(ctaMaps[b], m);
    uint32_t total;
    uint32_t e = rv_cta_scan(m, warpTot, &total) & 3u;             // the prefix applied to entry 0
    for (uint32_t b = lo; b < hi; b++) { entry[b] = (uint8_t)e; e = (ctaMaps[b] >> (2u * e)) & 3u; }
}

__global__ void __launch_bounds__(B2Z_RV_THREADS)
riscv_conv_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, uint64_t n, uint32_t startOffset, int enc, uint32_t unitLog,
                  const uint8_t* __restrict__ maps, const uint8_t* __restrict__ entry) {
    __shared__ __align__(16) uint8_t rows[B2Z_RV_THREADS * B2Z_RV_ROW];
    __shared__ uint32_t warpTot[B2Z_RV_THREADS / 32u];
    rv_stage(in, rows);
    const uint64_t chunk = (uint64_t)blockIdx.x * B2Z_RV_THREADS + threadIdx.x, base = chunk * B2Z_RV_CHUNK;
    const uint32_t m = base < n ? maps[chunk] : B2Z_RV_ID;
    uint32_t total;
    const uint32_t pre = rv_cta_scan(m, warpTot, &total);
    if (base >= n) return;
    uint64_t u0; uint32_t end; bool last;
    rv_chunk(base, n, unitLog, &u0, &end, &last);
    const uint8_t* row = rows + threadIdx.x * B2Z_RV_ROW;
    const uint32_t ia0 = startOffset + (uint32_t)(base - u0);
    uint8_t* dst = out + base;
    for (uint32_t p = 2u * ((pre >> (2u * entry[blockIdx.x])) & 3u); p < end;) {
        const uint32_t s = rv_step(row, p);
        if (s & 1u) {
            uint32_t w0 = rv_word(row, p), w1 = rv_word(row, p + 4u);
            if (enc) b2z_riscv_enc(&w0, &w1, ia0 + p); else b2z_riscv_dec(&w0, &w1, ia0 + p);
            for (uint32_t k = 0; k < 4u; k++) dst[p + k] = (uint8_t)(w0 >> (8u * k));
            if (s == 9u) for (uint32_t k = 0; k < 4u; k++) dst[p + 4u + k] = (uint8_t)(w1 >> (8u * k));
        }
        p += s & ~1u;
    }
}

}  // namespace b2z

#ifndef B2Z_CUEMU
// In place on a device buffer.  methodId: 7-Zip's filter ids (b2z_filter_ops.h); prop: delta distance (1..256) or the start offset
// ("pc") of the branch converters.  Branch converters leave a tail of n % 4 bytes untouched, like the reference (C/Bra.h:78-86).
// unitLog != 0 (encode only): the buffer is a run of independent units of 2^unitLog bytes -- the xz writer filters every Block on its own
int b2z_filter_units_device(b200z_ctx* ctx, uint32_t methodId, int encode, void* d_data, size_t n, uint32_t prop, uint32_t unitLog) {
    if (!ctx || (!d_data && n)) return B200Z_E_PARAM;
    if (unitLog && (!encode || unitLog < 12u)) return fail(ctx, B200Z_E_PARAM, "per-unit filtering is an encoder option (units >= 4 KiB)%s");
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    if (methodId == B200Z_F_DELTA) {
        if (prop < 1 || prop > 256) return fail(ctx, B200Z_E_PARAM, "delta distance must be 1..256%s");
        if (!n) return 0;
        if (encode) {
            if (ctx->batchStage.reserve(n)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
            CU(cudaMemcpyAsync(ctx->batchStage.p, d_data, n, cudaMemcpyDeviceToDevice, st));
            b2z::delta_enc_kernel<<<(unsigned)((n + 255) / 256 < 65535 ? (n + 255) / 256 : 65535), 256, 0, st>>>((const uint8_t*)ctx->batchStage.p, (uint8_t*)d_data, n, prop, unitLog);
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
        } else {
            const uint32_t rows = (65536u / prop) ? (65536u / prop) : 1u;
            const uint64_t tileBytes = (uint64_t)rows * prop;
            const uint32_t tiles = (uint32_t)((n + tileBytes - 1) / tileBytes);
            if (ctx->batchOff.reserve((size_t)tiles * prop + 64)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
            b2z::delta_colsum_kernel<<<tiles, 256, 0, st>>>((const uint8_t*)d_data, n, prop, rows, (uint8_t*)ctx->batchOff.p);
            b2z::delta_scan_kernel<<<1, 256, 0, st>>>((uint8_t*)ctx->batchOff.p, tiles, prop);
            b2z::delta_dec_kernel<<<tiles, 256, 0, st>>>((uint8_t*)d_data, n, prop, rows, (const uint8_t*)ctx->batchOff.p);
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 3;
        }
    } else if (methodId == B200Z_F_X86) {
        if (n >= 5) {
            if (ctx->batchStage.reserve(n)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
            CU(cudaMemcpyAsync(ctx->batchStage.p, d_data, n, cudaMemcpyDeviceToDevice, st));
            const uint64_t threads = (n + 31) / 32;
            b2z::x86_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, st>>>((const uint8_t*)ctx->batchStage.p, (uint8_t*)d_data, n, prop, encode, unitLog);
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
        }
    } else if (methodId == B200Z_F_ARMT) {
        if ((uintptr_t)d_data & 1u) return fail(ctx, B200Z_E_PARAM, "the Thumb converter needs a 2-byte aligned buffer%s");
        if (prop & 1u) return fail(ctx, B200Z_E_UNSUPPORTED, "start offset must be a multiple of the instruction size%s");
        const uint64_t nHalf = n >> 1;
        if (nHalf >= 2) {
            if (ctx->batchStage.reserve(n)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
            CU(cudaMemcpyAsync(ctx->batchStage.p, d_data, n, cudaMemcpyDeviceToDevice, st));
            b2z::armt_kernel<<<(unsigned)((nHalf + 255) / 256 < ctx->smCount * 64u ? (nHalf + 255) / 256 : ctx->smCount * 64u), 256, 0, st>>>((const uint16_t*)ctx->batchStage.p, (uint16_t*)d_data, nHalf, encode, prop, unitLog);
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
        }
    } else if (methodId == B200Z_F_ARM64 || methodId == B200Z_F_ARM || methodId == B200Z_F_PPC || methodId == B200Z_F_SPARC) {
        if ((uintptr_t)d_data & 3u) return fail(ctx, B200Z_E_PARAM, "branch converters need a 4-byte aligned buffer%s");
        if (prop & 3u) return fail(ctx, B200Z_E_UNSUPPORTED, "start offset must be a multiple of the instruction size%s");   // BranchMisc.cpp:57,99: E_INVALIDARG / E_NOTIMPL
        const uint64_t nWords = n >> 2;
        if (!nWords) return 0;
        b2z::bra_kernel<<<(unsigned)((nWords + 255) / 256 < ctx->smCount * 64u ? (nWords + 255) / 256 : ctx->smCount * 64u), 256, 0, st>>>((uint32_t*)d_data, nWords, methodId, encode, prop, unitLog);
        ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
    } else if (methodId == B200Z_F_RISCV) {
        if (prop & 1u) return fail(ctx, B200Z_E_UNSUPPORTED, "start offset must be a multiple of the instruction size%s");      // BranchMisc.cpp:57,99
        if (n >= 8) {                                               // (n & ~1) <= 6: nothing is scanned
            const uint64_t nChunks = (n + B2Z_RV_CHUNK - 1) / B2Z_RV_CHUNK, nCta = (nChunks + B2Z_RV_THREADS - 1) / B2Z_RV_THREADS;
            // the staged copy is read in whole CTA spans plus 8 look-ahead bytes; what lies past n is never looked at
            if (ctx->batchStage.reserve((size_t)nCta * B2Z_RV_SPAN + 64) || ctx->batchOff.reserve((size_t)(nCta * B2Z_RV_SPAN / B2Z_RV_CHUNK + 2 * nCta + 64)))
                return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
            CU(cudaMemcpyAsync(ctx->batchStage.p, d_data, n, cudaMemcpyDeviceToDevice, st));
            uint8_t* maps = (uint8_t*)ctx->batchOff.p;
            uint8_t* ctaMaps = maps + nCta * B2Z_RV_THREADS, *entry = ctaMaps + nCta;
            b2z::riscv_map_kernel<<<(unsigned)nCta, B2Z_RV_THREADS, 0, st>>>((const uint8_t*)ctx->batchStage.p, n, unitLog, maps, ctaMaps);
            b2z::riscv_scan_kernel<<<1, 1024, 0, st>>>(ctaMaps, entry, (uint32_t)nCta);
            b2z::riscv_conv_kernel<<<(unsigned)nCta, B2Z_RV_THREADS, 0, st>>>((const uint8_t*)ctx->batchStage.p, (uint8_t*)d_data, n, prop, encode, unitLog, maps, entry);
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 3;
        }
    } else return fail(ctx, B200Z_E_UNSUPPORTED, "filter not built on the GPU (BCJ2 / IA64)%s");
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(st));
    return 0;
}
extern "C" {

int b200z_filter_device(b200z_ctx* ctx, uint32_t methodId, int encode, void* d_data, size_t n, uint32_t prop) {
    return b2z_filter_units_device(ctx, methodId, encode, d_data, n, prop, 0);
}

int b200z_filter_host(b200z_ctx* ctx, uint32_t methodId, int encode, void* data, size_t n, uint32_t prop) {
    if (!ctx || (!data && n)) return B200Z_E_PARAM;
    CU(cudaSetDevice(ctx->device));
    if (ctx->dIn.reserve(n + 64)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
    if (n) CU(cudaMemcpyAsync(ctx->dIn.p, data, n, cudaMemcpyHostToDevice, ctx->stream));
    int rc = b200z_filter_device(ctx, methodId, encode, ctx->dIn.p, n, prop);
    if (rc) return rc;
    if (n) { CU(cudaMemcpyAsync(data, ctx->dIn.p, n, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream)); }
    ctx->stat[B200Z_S_H2D_BYTES] += (double)n; ctx->stat[B200Z_S_D2H_BYTES] += (double)n;
    return 0;
}

}  // extern "C"
#endif
