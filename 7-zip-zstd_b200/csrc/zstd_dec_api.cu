// zstd_dec_api.cu -- decoder half of the C ABI (include/b200z.h): drives stages D0..D3.
//
// Replaces the streaming loop of CPP/7zip/Compress/ZstdDecoder.cpp:108-173 (ZSTD_decompressStream
// over 128 KiB reads, frame after frame): here one call takes the whole Code() input, every frame
// of it (zstd or skippable) is located by the prepass and decoded in parallel.
#include "b2z_ctx.h"
#include <vector>

using namespace b2z;

static int dec_status_to_rc(b200z_ctx* ctx, uint32_t st) {
    if (st & B2Z_DERR_TABLE_FULL) return fail(ctx, B200Z_E_UNSUPPORTED, "more frames/blocks than the decoder tables hold%s");
    if (st & B2Z_DERR_UNSUPPORTED) return fail(ctx, B200Z_E_UNSUPPORTED, "dictionary or window > 1 GiB frames are not supported%s");
    if (st & B2Z_DERR_CORRUPT) return fail(ctx, B200Z_E_CORRUPT, "corrupt zstd data%s");          // a declared size that the blocks contradict is corruption, whatever else was noticed
    if (st & B2Z_DERR_DSTSIZE) return fail(ctx, B200Z_E_DSTSIZE, "destination too small%s");
    if (st & B2Z_DERR_CHECKSUM) return fail(ctx, B200Z_E_CHECKSUM, "content checksum mismatch%s");
    return 0;
}

// Sums what the blocks of a frame regenerate: raw / RLE blocks their size field, a compressed block `compressed` bytes
struct RegenSum {
    uint64_t* sum; uint32_t compressed;
    __host__ __device__ uint32_t operator()(uint32_t, uint32_t type, uint32_t bsize, uint64_t, uint32_t) const { *sum += type == 2 ? compressed : bsize; return 0; }
};

extern "C" {

// Walk frame headers (and block headers) on the host: cheap, sequential, no entropy decoding.
// Follows ZSTD_getFrameHeader / ZSTD_findFrameCompressedSize (C/zstd/zstd_decompress.c:482-600,702).
int b200z_zstd_frame_info(const void* srcv, size_t srcSize, uint64_t* contentSize, uint32_t* nFrames) {
    const HostBytes r{ (const uint8_t*)srcv, srcSize };
    uint64_t ip = 0, total = 0; uint32_t frames = 0; bool unknown = false;
    while (ip < srcSize) {
        if (srcSize - ip < 4) return B200Z_E_CORRUPT;
        const uint32_t magic = r.le32(ip);
        uint64_t sz;
        if (zstd_skippable(r, magic, ip, srcSize, &sz)) {
            if (srcSize - ip < sz) return B200Z_E_CORRUPT;
            ip += sz; continue;
        }
        if (magic != B2Z_ZSTD_MAGIC) return B200Z_E_CORRUPT;
        const ZstdFrameHdr h = zstd_frame_hdr(r, ip, srcSize);
        if (h.status) return B200Z_E_CORRUPT;
        uint64_t lower = 0;                                          // raw and RLE blocks: a lower bound where no size is declared
        const ZstdBlocks w = zstd_walk_blocks(r, ip, srcSize, h, RegenSum{ &lower, 0 });
        if (w.status) return B200Z_E_CORRUPT;
        if (h.fcsBytes) total += h.contentSize; else { total += lower; unknown = true; }
        frames++; ip = w.end;
    }
    if (nFrames) *nFrames = frames;
    if (contentSize) *contentSize = total;
    return unknown ? B200Z_E_UNSUPPORTED : B200Z_OK;
}


// The complete frames at the start of a buffer that may end inside a frame (streaming callers read the packed stream piece by
// piece).  *usedBytes = end of the last complete frame taken (skippable frames go with the frame that follows; trailing ones with
// the frame before), *contentBound = bytes those frames decode to -- exact where a frame declares its size, else the sum over its
// blocks of what a block can regenerate (raw / RLE: its size field, compressed: 128 KiB).  Stops before a frame that would take
// the sum past maxContent unless it is the first one.  B200Z_E_CORRUPT: the bytes at a frame start are no frame, or a frame's headers
// are malformed; the outputs still describe the complete frames in front of it.
int b200z_zstd_frame_prefix(const void* srcv, size_t srcSize, uint64_t maxContent, size_t* usedBytes, uint64_t* contentBound, uint32_t* nFrames) {
    const HostBytes r{ (const uint8_t*)srcv, srcSize };
    uint64_t ip = 0, total = 0; uint32_t frames = 0; size_t used = 0; int rc = B200Z_OK;
    while (ip < srcSize && srcSize - ip >= 4) {
        const uint32_t magic = r.le32(ip);
        uint64_t sz;
        if (zstd_skippable(r, magic, ip, srcSize, &sz)) {
            if (srcSize - ip < sz) break;
            ip += sz;
            if (frames) used = (size_t)ip;                          // after a frame: belongs to what was taken; before the first: to the frame to come
            continue;
        }
        if (magic != B2Z_ZSTD_MAGIC) { rc = B200Z_E_CORRUPT; break; }
        const ZstdFrameHdr h = zstd_frame_hdr(r, ip, srcSize);
        uint64_t bound = 0;
        const ZstdBlocks w = h.status ? ZstdBlocks{ 0, 0, h.status }
                                      : zstd_walk_blocks(r, ip, srcSize, h, RegenSum{ &bound, 131072u });
        if (w.status) { if (w.status == B2Z_DERR_CORRUPT) rc = B200Z_E_CORRUPT; break; }
        const uint64_t content = h.fcsBytes ? h.contentSize : bound;
        if (frames && total + content > maxContent) break;
        total += content; frames++; ip = w.end; used = (size_t)ip;
    }
    if (usedBytes) *usedBytes = used;
    if (contentBound) *contentBound = total;
    if (nFrames) *nFrames = frames;
    return rc;
}

}  // extern "C"

// hostDst != null: the output is also downloaded (after the execute kernel: every frame-warp is latency-bound and
// they all finish together, so splitting the download by frame groups only serialises the groups -- measured)
static int dec_impl(b200z_ctx* ctx, const void* d_src, size_t srcSize, void* d_dst, size_t dstCap, size_t* dstSize, void* hostDst) {
    if (!ctx || !dstSize || (!d_src && srcSize) || (!d_dst && dstCap)) return B200Z_E_PARAM;
    if ((uintptr_t)d_src & 7u) return fail(ctx, B200Z_E_PARAM, "device source must be 8-byte aligned%s");
    *dstSize = 0;
    if (!srcSize) return 0;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    // table capacities: frames >= 9 bytes each, blocks >= 3 bytes each; bounded to keep the tables small
    uint64_t frameCap = srcSize / 9 + 2; if (frameCap > (1u << 22)) frameCap = 1u << 22;
    uint64_t blockCap = srcSize / 3 + 2; { const uint64_t lim = srcSize / 128 + (1u << 20); if (blockCap > lim) blockCap = lim; }     // raw / RLE blocks cost a table entry only
    if (blockCap > 0x7FFFFFFFull) blockCap = 0x7FFFFFFFull;
    Arena& aFrames = ctx->decScratch[0]; Arena& aBlocks = ctx->decScratch[1]; Arena& aCounts = ctx->decScratch[2];
    Arena& aLits = ctx->decScratch[3]; Arena& aSeqs = ctx->decScratch[4];
    if (aFrames.reserve(frameCap * sizeof(DecFrame)) || aBlocks.reserve(blockCap * sizeof(DecBlock)) || aCounts.reserve(64))
        return fail(ctx, B200Z_E_MEMORY, "decoder table allocation failed%s");
    DecFrame* frames = (DecFrame*)aFrames.p; DecBlock* blocks = (DecBlock*)aBlocks.p;
    DecCounts* counts = (DecCounts*)aCounts.p; uint64_t* total = (uint64_t*)((uint8_t*)aCounts.p + 40);
    CU(cudaEventRecord(ctx->ev[0], st));
    DecCounts hc;
    static_assert(sizeof(DecCounts) == 40, "DecCounts is fetched as five words");
    // stage D0, first with mcmilk's size hints trusted (one hop per frame); a stream that then fails to index -- a skippable frame that only
    // looks like a hint -- is walked again block header by block header, as the reference does for every stream
    for (int pass = 0; pass < 2; pass++) {
        CU(cudaMemsetAsync(aCounts.p, 0, 64, st));
        launch_zstd_dec_find_frames((const uint8_t*)d_src, srcSize, frames, (uint32_t)frameCap, counts, pass == 0, st);
        CU(cudaGetLastError());
        { const int frc = b2z_fetch_small(ctx, &hc, counts, sizeof(hc), st); if (frc) return frc; }
        const uint32_t hinted = hc.nUnits;
        ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
        if (!hc.status) {
            launch_zstd_dec_index_blocks((const uint8_t*)d_src, srcSize, frames, hc.nFrames, blocks, (uint32_t)blockCap, counts, st);
            CU(cudaGetLastError());
            { const int frc = b2z_fetch_small(ctx, &hc, counts, sizeof(hc), st); if (frc) return frc; }
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 3;
        }
        if (!hc.status || !hinted || (hc.status & ~B2Z_DERR_CORRUPT)) break;       // fine, or not the hints' fault
    }
    CU(cudaEventRecord(ctx->ev[3], st));
    if (hc.status) return dec_status_to_rc(ctx, hc.status);
    if (aLits.reserve((size_t)hc.nSlots * 131072ull + 64) || aSeqs.reserve((size_t)hc.nSlots * B2Z_DEC_MAXSEQ * 8ull + 64) ||
        ctx->decScratch[5].reserve(zstd_dec_entropy_scratch_bytes(hc.nBlocks) + zstd_dec_unit_state_bytes(hc.nFrames, hc.nBlocks) + 64))
        return fail(ctx, B200Z_E_MEMORY, "decoder scratch allocation failed (input too large for one pass)%s");
    launch_zstd_dec_entropy((const uint8_t*)d_src, srcSize, blocks, hc.nBlocks, (uint8_t*)aLits.p, (uint64_t*)aSeqs.p, ctx->decScratch[5].p, ctx->smCount, st, st, ctx->ev[4], ctx->ev[5]);
    CU(cudaGetLastError());
    CU(cudaEventRecord(ctx->ev[1], st));
    // stage J (zstd_dec.cu): frames whose units would form one chain -- what the reference's encoder writes -- are resolved by pointer
    // jumping.  Only a stream with a frame of enough blocks pays for the extra look at the counters.
    const uint32_t jumpMode = (uint32_t)ctx->decJump;
    const bool maybeJump = jumpMode == 2u || (jumpMode == 1u && (hc.maxFrameBlocks + B2Z_DEC_UNIT_BLOCKS - 1u) / B2Z_DEC_UNIT_BLOCKS >= B2Z_DEC_JUMP_MIN_UNITS);
    launch_zstd_dec_layout(frames, hc.nFrames, blocks, dstCap, counts, total, maybeJump ? jumpMode : 0u, st);
    CU(cudaGetLastError());
    if (maybeJump) {
        struct { DecCounts c; uint64_t total; } hj;
        { const int frc = b2z_fetch_small(ctx, &hj, counts, 48, st); if (frc) return frc; }
        if (hj.c.status) return dec_status_to_rc(ctx, hj.c.status);
        if (hj.c.nJump) {
            Arena& aPtr = ctx->decScratch[8];
            const uint32_t segLog = ctx->decJumpSegLog;
            if (aPtr.reserve(zstd_dec_jump_scratch_bytes(hj.total, segLog))) return fail(ctx, B200Z_E_MEMORY, "decoder scratch allocation failed (stage J pointers)%s");
            launch_zstd_dec_jump((const uint8_t*)d_src, frames, hc.nFrames, blocks, hc.nBlocks, (const uint8_t*)aLits.p, (const uint64_t*)aSeqs.p,
                                 (uint8_t*)d_dst, hj.total, segLog, counts, aPtr.p, ctx->smCount, st);
            CU(cudaGetLastError());
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += (2 + B2Z_DEC_JUMP_ROUNDS) * ((hj.total + (1ull << segLog) - 1) >> segLog);
            ctx->stat[B200Z_S_DEC_JUMP_FRAMES] += hj.c.nJump;
        }
    }
    uint32_t* unitState = (uint32_t*)((uint8_t*)ctx->decScratch[5].p + ((zstd_dec_entropy_scratch_bytes(hc.nBlocks) + 15u) & ~(size_t)15u));   // behind D1's scratch
    launch_zstd_dec_exec((const uint8_t*)d_src, frames, hc.nFrames, blocks, hc.nBlocks, (const uint8_t*)aLits.p, (const uint64_t*)aSeqs.p,
                         (uint8_t*)d_dst, counts, unitState, ctx->smCount, st);
    CU(cudaGetLastError());
    launch_zstd_dec_verify((const uint8_t*)d_src, frames, hc.nFrames, (const uint8_t*)d_dst, counts, st);
    CU(cudaGetLastError());
    CU(cudaEventRecord(ctx->ev[2], st));
    struct { DecCounts c; uint64_t total; } hr;                                // counts at +0, the total at +40 of the same 64-byte scratch
    { const int frc = b2z_fetch_small(ctx, &hr, counts, 48, st); if (frc) return frc; }
    ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 7;
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[3]); ctx->stat[B200Z_S_DEC_PREPASS_MS] += ms;
    cudaEventElapsedTime(&ms, ctx->ev[3], ctx->ev[1]); ctx->stat[B200Z_S_DEC_ENTROPY_MS] += ms;
    cudaEventElapsedTime(&ms, ctx->ev[1], ctx->ev[2]); ctx->stat[B200Z_S_DEC_EXEC_MS] += ms;
    if (hr.c.status) return dec_status_to_rc(ctx, hr.c.status);
    if (hostDst && hr.total) { CU(cudaMemcpyAsync(hostDst, d_dst, hr.total, cudaMemcpyDeviceToHost, st)); CU(cudaStreamSynchronize(st)); ctx->stat[B200Z_S_D2H_BYTES] += (double)hr.total; }
    *dstSize = (size_t)hr.total;
    return 0;
}

extern "C" {

int b200z_zstd_decompress_device(b200z_ctx* ctx, const void* d_src, size_t srcSize, void* d_dst, size_t dstCap, size_t* dstSize) {
    return dec_impl(ctx, d_src, srcSize, d_dst, dstCap, dstSize, nullptr);
}

// Host-side split of a compressed stream into batches of whole frames (only when every frame declares its
// content size): returns false if the stream cannot be split that way (the caller then decodes in one shot).
static bool split_frames(const uint8_t* src, size_t srcSize, uint64_t targetOut, std::vector<HostBatch>& out) {
    const HostBytes r{ src, srcSize };
    size_t ip = 0; HostBatch cur{0, 0, 0, true};
    while (ip < srcSize) {
        if (srcSize - ip < 4) return false;
        const uint32_t magic = r.le32(ip);
        uint64_t sz;
        if (zstd_skippable(r, magic, ip, srcSize, &sz)) {
            if (srcSize - ip < sz) return false;
            ip += sz; continue;                                      // hints/skippable data stay attached to the following frame
        }
        if (magic != B2Z_ZSTD_MAGIC) return false;
        const ZstdFrameHdr h = zstd_frame_hdr(r, ip, srcSize);
        if (h.status || !h.fcsBytes) return false;
        const ZstdBlocks w = zstd_walk_blocks(r, ip, srcSize, h, ZstdEmitNone{});
        if (w.status) return false;
        ip = w.end;
        cur.srcLen = ip - cur.srcOff; cur.outSize += h.contentSize;
        if (cur.outSize >= targetOut) { out.push_back(cur); cur = HostBatch{ ip, 0, 0, true }; }
    }
    if (cur.srcLen || cur.outSize) { cur.srcLen = srcSize - cur.srcOff; out.push_back(cur); }
    else if (!out.empty()) out.back().srcLen = srcSize - out.back().srcOff;
    return true;
}

// Host-pointer decompress: batches of whole frames flow through the pipeline of b2z_host_pipeline.  Every batch knows where its
// output goes (the frames declare their sizes), so devices never wait for each other.
int b200z_zstd_decompress_host(b200z_ctx* ctx, const void* src, size_t srcSize, void* dst, size_t dstCap, size_t* dstSize) {
    if (!ctx || !dstSize || (!src && srcSize) || (!dst && dstCap)) return B200Z_E_PARAM;
    *dstSize = 0;
    if (!srcSize) return 0;
    CU(cudaSetDevice(ctx->device));
    std::vector<HostBatch> batches;
    const size_t nDev = 1 + ctx->peers.size();
    uint64_t target = 1ull << ctx->hostBatchLog;                     // decoded bytes per batch
    if (nDev > 1) { const uint64_t per = (uint64_t)srcSize * 3 / (2 * nDev) + 1; if (per < target) target = per; }   // about two batches per device (packed size x 3 ~ output)
    if ((nDev == 1 && srcSize <= (target >> 2)) || !split_frames((const uint8_t*)src, srcSize, target, batches) || (batches.size() < 2 && nDev == 1) || batches.empty()) {
        // one shot
        if (ctx->dIn.reserve(srcSize + 64) || ctx->dOut.reserve(dstCap + 64)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
        CU(cudaMemcpyAsync(ctx->dIn.p, src, srcSize, cudaMemcpyHostToDevice, ctx->stream));
        ctx->stat[B200Z_S_H2D_BYTES] += (double)srcSize;
        size_t out = 0;
        int rc = dec_impl(ctx, ctx->dIn.p, srcSize, ctx->dOut.p, dstCap, &out, dst);
        if (rc) return rc;
        *dstSize = out;
        return 0;
    }
    size_t maxIn = 0; uint64_t maxOut = 0, total = 0;
    for (const HostBatch& b : batches) { if (b.srcLen > maxIn) maxIn = b.srcLen; if (b.outSize > maxOut) maxOut = b.outSize; total += b.outSize; }
    if (total > dstCap) return fail(ctx, B200Z_E_DSTSIZE, "destination too small%s");
    const size_t inStride = (maxIn + 64 + 255) & ~(size_t)255, outStride = ((size_t)maxOut + 64 + 255) & ~(size_t)255;
    const int rc = b2z_host_pipeline(ctx, (const uint8_t*)src, (uint8_t*)dst, batches, inStride, outStride, [&](b200z_ctx* c, size_t i, const uint8_t* dIn, uint8_t* dOut, uint64_t* out) {
        size_t n = 0;
        const int drc = dec_impl(c, dIn, batches[i].srcLen, dOut, (size_t)batches[i].outSize, &n, nullptr);
        if (drc) return drc;
        if (n != batches[i].outSize) return fail(c, B200Z_E_CORRUPT, "frame content size mismatch%s");
        *out = n;
        return 0;
    }, &total);
    if (rc) return rc;
    *dstSize = (size_t)total;
    return 0;
}

}  // extern "C"
