// lzma2_api.cu -- C ABI, LZMA2 (method 21) decoder side.  See include/b200z.h for the reference interfaces replaced.
#include <vector>
#include "b2z_ctx.h"
#include "b2z_lzma2.h"

using namespace b2z;

namespace {
struct Lz2EmitNone { __host__ __device__ void operator()(uint32_t, uint64_t, uint64_t, uint64_t, uint64_t) const {} };

int lz2_status_to_rc(b200z_ctx* ctx, uint32_t status) {
    if (status & 2u) return fail(ctx, B200Z_E_UNSUPPORTED, "LZMA2: a single dictionary-reset block of 4 GiB or more%s");
    return fail(ctx, B200Z_E_CORRUPT, "LZMA2: malformed stream%s");
}
}  // namespace

extern "C" {

int b200z_lzma2_stream_info(const void* src, size_t srcSize, uint64_t* contentSize, uint32_t* nBlocks, size_t* srcUsed) {
    if (!src && srcSize) return B200Z_E_PARAM;
    Lz2Counts c;
    lzma2_walk((const uint8_t*)src, srcSize, c, Lz2EmitNone{});
    if (contentSize) *contentSize = c.total;
    if (nBlocks) *nBlocks = c.nBlocks;
    if (srcUsed) *srcUsed = (size_t)c.srcUsed;
    if (c.status & 2u) return B200Z_E_UNSUPPORTED;
    return c.status ? B200Z_E_CORRUPT : B200Z_OK;
}

// The complete dictionary-reset blocks at the start of a buffer that may end inside a chunk (streaming callers).  A block is
// known to be complete once the header of the next reset chunk, or the end marker, has been seen.  *usedBytes = offset of that
// boundary (past the end marker when *ended), *contentSize = decoded bytes of the blocks before it.  Stops at the first boundary
// at or beyond maxContent.  The caller decodes [0, usedBytes) -- appending the 0x00 end marker when !*ended -- and goes on from there.
int b200z_lzma2_stream_prefix(const void* srcv, size_t srcSize, uint64_t maxContent, size_t* usedBytes, uint64_t* contentSize, uint32_t* nBlocks, int* ended) {
    const uint8_t* src = (const uint8_t*)srcv;
    uint64_t ip = 0, total = 0, boundary = 0, boundaryTotal = 0;
    uint32_t nb = 0, nbAtBoundary = 0, needInit = 0xE0;
    int end = 0, rc = B200Z_OK;
    while (ip < srcSize) {
        const Lz2Chunk ch = lzma2_chunk(src + ip, srcSize - ip, needInit);
        if (ch.status) { if (ch.status == B2Z_DERR_CORRUPT) rc = B200Z_E_CORRUPT; break; }         // cut off: wait for more bytes
        if (ch.kind == LZ2_CHUNK_END) { boundary = ip + 1; boundaryTotal = total; nbAtBoundary = nb; end = 1; break; }
        if (ch.reset) {                                         // everything before this header is whole blocks
            boundary = ip; boundaryTotal = total; nbAtBoundary = nb; nb++;
            if (nbAtBoundary && boundaryTotal >= maxContent) break;
        }
        if (ch.hdr + ch.pack > srcSize - ip) break;
        total += ch.unpack; ip += ch.hdr + ch.pack;
    }
    if (usedBytes) *usedBytes = (size_t)boundary;
    if (contentSize) *contentSize = boundaryTotal;
    if (nBlocks) *nBlocks = nbAtBoundary;
    if (ended) *ended = end;
    return rc;
}

int b200z_lzma2_decompress_device(b200z_ctx* ctx, const void* d_src, size_t srcSize, uint32_t dictProp,
                                  void* d_dst, size_t dstCap, size_t* dstSize) {
    if (!ctx || !dstSize || (!d_src && srcSize) || (!d_dst && dstCap)) return B200Z_E_PARAM;
    *dstSize = 0;
    if (dictProp > 40) return fail(ctx, B200Z_E_UNSUPPORTED, "LZMA2: dictionary property above 40%s");
    if (!srcSize) return fail(ctx, B200Z_E_CORRUPT, "LZMA2: empty stream (no end marker)%s");
    const uint32_t dictSize = lzma2_dict_size(dictProp);
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    Arena& aBlocks = ctx->decScratch[6]; Arena& aCounts = ctx->decScratch[7];
    uint64_t cap = srcSize / 65536 + 1024;                      // typical: far fewer blocks than chunks; re-run if it overflows
    if (aCounts.reserve(64)) return fail(ctx, B200Z_E_MEMORY, "LZMA2: table allocation failed%s");
    Lz2Counts* counts = (Lz2Counts*)aCounts.p;
    Lz2Counts hc;
    CU(cudaEventRecord(ctx->ev[0], st));
    for (int pass = 0; pass < 2; pass++) {
        if (aBlocks.reserve(cap * sizeof(Lz2Block))) return fail(ctx, B200Z_E_MEMORY, "LZMA2: table allocation failed%s");
        launch_lzma2_walk((const uint8_t*)d_src, srcSize, (Lz2Block*)aBlocks.p, (uint32_t)cap, counts, st);
        CU(cudaGetLastError());
        { const int frc = b2z_fetch_small(ctx, &hc, counts, sizeof(hc), st); if (frc) return frc; }
        ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
        if (hc.status) return lz2_status_to_rc(ctx, hc.status);
        if (hc.nBlocks <= cap) break;
        cap = hc.nBlocks;
    }
    if (hc.total > dstCap) return fail(ctx, B200Z_E_DSTSIZE, "destination too small%s");
    CU(cudaEventRecord(ctx->ev[3], st));
    const int mode = ctx->lz2Mode == 3 ? 0 : ctx->lz2Mode;          // (3 is an encoder-only choice)
    uint16_t* spill = nullptr;
    if (mode != 1 && hc.nBlocks > 13u * ctx->smCount / 2u) {          // worth leaving shared memory only with many blocks
        if (ctx->decScratch[5].reserve(lzma2_lit_spill_bytes(hc.nBlocks, hc.maxLcLp)) == 0) spill = (uint16_t*)ctx->decScratch[5].p;
    }
    if (mode == 2 && !spill) {
        if (ctx->decScratch[5].reserve(lzma2_lit_spill_bytes(hc.nBlocks, hc.maxLcLp))) return fail(ctx, B200Z_E_MEMORY, "LZMA2: model allocation failed%s");
        spill = (uint16_t*)ctx->decScratch[5].p;
    }
    CU(launch_lzma2_decode((const uint8_t*)d_src, (const Lz2Block*)aBlocks.p, hc.nBlocks, hc.maxLcLp, dictSize, (uint8_t*)d_dst, counts,
                           spill, ctx->smCount, mode, st));
    CU(cudaEventRecord(ctx->ev[2], st));
    { const int frc = b2z_fetch_small(ctx, &hc, counts, sizeof(hc), st); if (frc) return frc; }
    ctx->stat[B200Z_S_KERNEL_LAUNCHES] += hc.nBlocks ? 1 : 0;
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[3]); ctx->stat[B200Z_S_DEC_PREPASS_MS] += ms;
    cudaEventElapsedTime(&ms, ctx->ev[3], ctx->ev[2]); ctx->stat[B200Z_S_DEC_ENTROPY_MS] += ms;
    if (hc.status) return lz2_status_to_rc(ctx, hc.status);
    *dstSize = (size_t)hc.total;
    return 0;
}

// Host-pointer form: upload, decode, download (the packed stream is small next to its output; the download dominates).
int b200z_lzma2_decompress_host(b200z_ctx* ctx, const void* src, size_t srcSize, uint32_t dictProp,
                                void* dst, size_t dstCap, size_t* dstSize) {
    if (!ctx || !dstSize || (!src && srcSize) || (!dst && dstCap)) return B200Z_E_PARAM;
    *dstSize = 0;
    uint64_t total = 0; size_t used = 0;
    int rc = b200z_lzma2_stream_info(src, srcSize, &total, nullptr, &used);        // headers only: rejects garbage before any upload
    if (rc) return rc == B200Z_E_UNSUPPORTED ? lz2_status_to_rc(ctx, 2u) : lz2_status_to_rc(ctx, 1u);
    if (total > dstCap) return fail(ctx, B200Z_E_DSTSIZE, "destination too small%s");
    CU(cudaSetDevice(ctx->device));
    if (ctx->dIn.reserve(used + 64) || ctx->dOut.reserve((size_t)total + 64)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
    CU(cudaMemcpyAsync(ctx->dIn.p, src, used, cudaMemcpyHostToDevice, ctx->stream));
    ctx->stat[B200Z_S_H2D_BYTES] += (double)used;
    size_t out = 0;
    rc = b200z_lzma2_decompress_device(ctx, ctx->dIn.p, used, dictProp, ctx->dOut.p, (size_t)total, &out);
    if (rc) return rc;
    if (out) { CU(cudaMemcpyAsync(dst, ctx->dOut.p, out, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream)); }
    ctx->stat[B200Z_S_D2H_BYTES] += (double)out;
    *dstSize = out;
    return 0;
}

}  // extern "C"
