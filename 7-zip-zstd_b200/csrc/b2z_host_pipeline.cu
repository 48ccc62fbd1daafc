// b2z_host_pipeline.cu -- the batch pipeline shared by the host-pointer entry points (b2z_ctx.h): zstd and LZMA2 compress, zstd
// decompress.  Batches of whole frames are dealt round-robin to the devices of a context; every device runs H2D | kernels | D2H over its
// batches on its own host thread, streams and staging, so PCIe time hides under kernel time when the host buffers are pinned.  The
// ordered output mirrors ZSTDMT_flushProduced (zstdmt_compress.c:1488).
#include <mutex>
#include <thread>
#include <condition_variable>
#include "b2z_ctx.h"

namespace {

struct Pipe {
    const uint8_t* src = nullptr; uint8_t* dst = nullptr; const std::vector<HostBatch>* batches = nullptr; size_t inStride = 0, outStride = 0;
    const HostCode* code = nullptr;
    std::mutex m; std::condition_variable cv;
    std::vector<uint64_t> size; std::vector<char> known;         // output bytes of every batch, once known
    int rc = 0; b200z_ctx* errCtx = nullptr;                     // first error
    void fail_with(int code, b200z_ctx* c) { std::lock_guard<std::mutex> g(m); if (!rc) { rc = code; errCtx = c; } cv.notify_all(); }
    bool failed() { std::lock_guard<std::mutex> g(m); return rc != 0; }
    void publish(size_t i, uint64_t n) { std::lock_guard<std::mutex> g(m); size[i] = n; known[i] = 1; cv.notify_all(); }
    // output offset of batch i: blocks until the sizes of batches 0 .. i-1 are known; false when another worker failed
    bool offset_of(size_t i, uint64_t* off) {
        std::unique_lock<std::mutex> g(m);
        uint64_t sum = 0;
        for (size_t k = 0; k < i; k++) { cv.wait(g, [&] { return rc != 0 || known[k]; }); if (rc) return false; sum += size[k]; }
        *off = sum; return true;
    }
};

// one worker's share: batches first, first + stride, ...  pe[0..1]: input of buffer b uploaded; pe[2..3]: output of buffer b downloaded
int pipe_run(b200z_ctx* ctx, Pipe* p, size_t first, size_t stride) {
    CU(cudaSetDevice(ctx->device));
    const std::vector<HostBatch>& B = *p->batches;
    if (ctx->dIn.reserve(2 * p->inStride) || ctx->dOut.reserve(2 * p->outStride)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
    uint8_t* dIn[2] = { (uint8_t*)ctx->dIn.p, (uint8_t*)ctx->dIn.p + p->inStride };
    uint8_t* dOut[2] = { (uint8_t*)ctx->dOut.p, (uint8_t*)ctx->dOut.p + p->outStride };
    CU(cudaMemcpyAsync(dIn[0], p->src + B[first].srcOff, B[first].srcLen, cudaMemcpyHostToDevice, ctx->stream2));
    CU(cudaEventRecord(ctx->pe[0], ctx->stream2));
    size_t k = 0;
    for (size_t i = first; i < B.size(); i += stride, k++) {
        const int b = (int)(k & 1);
        if (p->failed()) return 0;                                           // another worker failed: its error is the call's
        if (i + stride < B.size()) {                                         // upload the next batch while this one is coded
            // its buffer was last read by the kernels of the batch before this one, which have been synchronised already
            const HostBatch& nx = B[i + stride];
            CU(cudaMemcpyAsync(dIn[b ^ 1], p->src + nx.srcOff, nx.srcLen, cudaMemcpyHostToDevice, ctx->stream2));
            CU(cudaEventRecord(ctx->pe[b ^ 1], ctx->stream2));
        }
        CU(cudaStreamWaitEvent(ctx->stream, ctx->pe[b], 0));                 // input there
        if (k >= 2) CU(cudaStreamWaitEvent(ctx->stream, ctx->pe[2 + b], 0)); // output buffer drained
        uint64_t out = 0;
        const int rc = (*p->code)(ctx, i, dIn[b], dOut[b], &out);
        if (rc) return rc;
        p->publish(i, out);
        uint64_t off = 0;
        if (!p->offset_of(i, &off)) return 0;
        if (out) CU(cudaMemcpyAsync(p->dst + off, dOut[b], out, cudaMemcpyDeviceToHost, ctx->stream3));
        CU(cudaEventRecord(ctx->pe[2 + b], ctx->stream3));
        ctx->stat[B200Z_S_H2D_BYTES] += (double)B[i].srcLen; ctx->stat[B200Z_S_D2H_BYTES] += (double)out;
    }
    return 0;
}

void pipe_worker(b200z_ctx* ctx, Pipe* p, size_t first, size_t stride) {
    int rc = pipe_run(ctx, p, first, stride);
    // every exit waits for this worker's copies: once the call has returned, none may still read src or write dst
    const cudaError_t e2 = cudaStreamSynchronize(ctx->stream2), e3 = cudaStreamSynchronize(ctx->stream3);
    if (!rc && (e2 != cudaSuccess || e3 != cudaSuccess)) {
        cudaGetLastError();
        rc = fail(ctx, B200Z_E_CUDA, "host pipeline copy: %s", cudaGetErrorString(e2 != cudaSuccess ? e2 : e3));
    }
    if (rc) p->fail_with(rc, ctx);
}

}  // namespace

int b2z_host_pipeline(b200z_ctx* ctx, const uint8_t* src, uint8_t* dst, const std::vector<HostBatch>& batches, size_t inStride, size_t outStride,
                      const HostCode& code, uint64_t* total) {
    Pipe p; p.src = src; p.dst = dst; p.batches = &batches; p.inStride = inStride; p.outStride = outStride; p.code = &code;
    p.size.assign(batches.size(), 0); p.known.assign(batches.size(), 0);
    for (size_t i = 0; i < batches.size(); i++) if (batches[i].outKnown) { p.size[i] = batches[i].outSize; p.known[i] = 1; }
    const size_t nDev = 1 + ctx->peers.size(), nWorkers = nDev < batches.size() ? nDev : batches.size();
    std::vector<std::thread> threads;
    for (size_t d = 1; d < nWorkers; d++) threads.emplace_back(pipe_worker, ctx->peers[d - 1], &p, d, nWorkers);
    if (nWorkers) pipe_worker(ctx, &p, 0, nWorkers);
    for (std::thread& t : threads) t.join();
    if (p.rc) { if (p.errCtx && p.errCtx != ctx) snprintf(ctx->err, sizeof(ctx->err), "device %d: %.200s", p.errCtx->device, p.errCtx->err); return p.rc; }
    uint64_t sum = 0; for (uint64_t v : p.size) sum += v;
    *total = sum;
    return 0;
}
