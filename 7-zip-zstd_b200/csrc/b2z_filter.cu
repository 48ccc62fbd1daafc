// b2z_filter.cu -- the pre/post filters that sit in front of the main coder in a 7z folder or an xz filter chain, on the GPU
// (SURVEY.md 8(f) item 3): Delta and the stateless branch converters ARM64, ARM, PPC, SPARC.  In place on a device buffer.
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
//   not here       BCJ2 (four output streams + a range coder), RISCV, IA64 -- left to the host.
// Oracle statement: oracle/filter_oracle.c; both are checked against the reference's functions (oracle/_ref/libref_xz.so).
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
    } else return fail(ctx, B200Z_E_UNSUPPORTED, "filter not built on the GPU (BCJ2 / RISCV / IA64)%s");
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
