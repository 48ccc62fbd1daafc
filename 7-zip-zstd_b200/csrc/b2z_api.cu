// b2z_api.cu -- the extern "C" shim of libb200z.so (see include/b200z.h).
//
// Host dispatcher for one device: owns the stream, the scratch arenas (candidate words, per-block
// sequence/literal/slot arrays) and the staging buffers of the host-pointer entry points.
// Replaces the job/worker plumbing of C/zstd/zstdmt_compress.c (ZSTDMT_compressStream_generic
// :1853, ZSTDMT_createCompressionJob :1403, ZSTDMT_flushProduced :1488): frames are the jobs,
// warps are the workers, the assemble kernels are the ordered flush.
#include <vector>
#include "b2z_ctx.h"
#include "b2z_lzma2.h"
#include "b2z_lzma_model.h"

using namespace b2z;

__global__ void b2z_store_small_kernel(uint64_t* __restrict__ hostDst, const uint64_t* __restrict__ src, uint32_t nWords) {
    if (threadIdx.x < nWords) hostDst[threadIdx.x] = src[threadIdx.x];
    __threadfence_system();
}
int b2z_fetch_small(b200z_ctx* ctx, void* hostDst, const void* d_src, size_t bytes, cudaStream_t st) {
    if (bytes > 256 || (bytes & 7u)) return fail(ctx, B200Z_E_PARAM, "b2z_fetch_small: size%s");
    if (!ctx->hostSmall && cudaHostAlloc((void**)&ctx->hostSmall, 256, cudaHostAllocMapped) != cudaSuccess) { cudaGetLastError(); return fail(ctx, B200Z_E_MEMORY, "pinned allocation failed%s"); }
    b2z_store_small_kernel<<<1, 32, 0, st>>>(ctx->hostSmall, (const uint64_t*)d_src, (uint32_t)(bytes / 8));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(st));
    memcpy(hostDst, ctx->hostSmall, bytes);
    return 0;
}

extern "C" {

int b200z_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int b200z_create(b200z_ctx** out, int device) {
    if (!out) return B200Z_E_PARAM;
    *out = nullptr;
    int n = b200z_device_count();
    if (n <= 0 || device < 0 || device >= n) return B200Z_E_NODEVICE;   // no CPU fallback, by design
    b200z_ctx* ctx = new (std::nothrow) b200z_ctx();
    if (!ctx) return B200Z_E_MEMORY;
    ctx->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return B200Z_E_NODEVICE; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->smCount = (uint32_t)prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return B200Z_E_CUDA; }
    if (cudaStreamCreateWithFlags(&ctx->stream2, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return B200Z_E_CUDA; }
    if (cudaStreamCreateWithFlags(&ctx->stream3, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return B200Z_E_CUDA; }
    for (int i = 0; i < 4; i++) cudaEventCreateWithFlags(&ctx->pe[i], cudaEventDisableTiming);
    for (int i = 0; i < 8; i++) cudaEventCreate(&ctx->ev[i]);
    ctx->geom.frameLog = B2Z_DEF_FRAMELOG; ctx->geom.hashLogL = B2Z_DEF_HASHLOG_L; ctx->geom.hashLogS = B2Z_DEF_HASHLOG_S;
    ctx->geom.chunkLog = B2Z_DEF_CHUNKLOG; ctx->geom.regionLog = B2Z_DEF_PLAIN_REGIONLOG;
    ctx->geom.windowLog = B2Z_DEF_FRAMELOG; ctx->geom.flags = 1u | (B2Z_DEF_LZ2_SLICELOG << 8);   // size hints on: lets any decoder (ours included) find frames without walking blocks
    *out = ctx;
    return B200Z_OK;
}

// One context over several devices: the host-pointer entry points (what ICompressCoder::Code() calls) cut their input into
// batches of whole frames and deal them round-robin to the devices, each with its own streams, staging and scratch; the output is
// written in input order and does not depend on the device count.  The role of ZSTDMT_createCompressionJob / ZSTDMT_flushProduced
// (zstdmt_compress.c:1403,1488) and MtCoder_Code (MtCoder.c:445) one level up: devices are the workers.
int b200z_create_multi(b200z_ctx** out, const int* devices, int nDevices) {
    if (!out || !devices || nDevices < 1) return B200Z_E_PARAM;
    *out = nullptr;
    // (a device may be listed more than once: each entry is a worker with its own streams and scratch)
    b200z_ctx* first = nullptr;
    int rc = b200z_create(&first, devices[0]);
    if (rc) return rc;
    for (int i = 1; i < nDevices; i++) {
        b200z_ctx* p = nullptr;
        rc = b200z_create(&p, devices[i]);
        if (rc) { b200z_destroy(first); return rc; }
        first->peers.push_back(p);
    }
    *out = first;
    return B200Z_OK;
}

int b200z_device_list(b200z_ctx* ctx, int* devices, int cap) {
    if (!ctx) return 0;
    const int n = 1 + (int)ctx->peers.size();
    for (int i = 0; i < n && i < cap && devices; i++) devices[i] = i == 0 ? ctx->device : ctx->peers[(size_t)i - 1]->device;
    return n;
}

void b200z_destroy(b200z_ctx* ctx) {
    if (!ctx) return;
    for (b200z_ctx* p : ctx->peers) b200z_destroy(p);
    ctx->peers.clear();
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    Arena* all[] = { &ctx->tables, &ctx->seqs, &ctx->nseq, &ctx->lits, &ctx->nlit, &ctx->slots, &ctx->slotSize,
                     &ctx->blockOff, &ctx->frameOff, &ctx->scalars, &ctx->dIn, &ctx->dOut, &ctx->cks, &ctx->ready, &ctx->batchStage, &ctx->batchOff, &ctx->batchSize, &ctx->cand, &ctx->choice, &ctx->crcOff, &ctx->crcLen, &ctx->crcOut };
    for (Arena* a : all) a->release();
    for (Arena& a : ctx->decScratch) a.release();
    for (int i = 0; i < 8; i++) if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
    if (ctx->stream3) cudaStreamDestroy(ctx->stream3);
    for (int i = 0; i < 4; i++) if (ctx->pe[i]) cudaEventDestroy(ctx->pe[i]);
    if (ctx->hostOne) cudaFreeHost(ctx->hostOne);
    if (ctx->hostSmall) cudaFreeHost(ctx->hostSmall);
    delete ctx;
}

static int set_param_one(b200z_ctx* ctx, int param, int64_t v);
int b200z_set_param(b200z_ctx* ctx, int param, int64_t v) {
    if (!ctx) return B200Z_E_PARAM;
    const int rc = set_param_one(ctx, param, v);
    if (rc == 0) for (b200z_ctx* p : ctx->peers) set_param_one(p, param, v);         // every device of the group codes with the same parameters
    return rc;
}
static int set_param_one(b200z_ctx* ctx, int param, int64_t v) {
    switch (param) {
    case B200Z_P_LEVEL:     if (v < 1 || v > 22) return fail(ctx, B200Z_E_PARAM, "level out of range%s"); ctx->level = (int)v;
                            // levels 1-7: the level-3-class greedy/lazy stage M; 8-22: the price-based stage C + stage Z
                            ctx->geom.flags = (ctx->geom.flags & ~(B2Z_FLAG_ZSTD_OPT | B2Z_FLAG_FIND_FAST | B2Z_FLAG_FIND_STEP)) | (v >= B2Z_ZSTD_OPT_LEVEL ? B2Z_FLAG_ZSTD_OPT : 0u) | b2z_level_find_flags((int)v);
                            // the level ladder of stage F (b2z_params.h): 1-2 the short table alone, in the long table's room; 3-4 both; 5-7 both + same-step lanes
                            ctx->geom.hashLogL = B2Z_DEF_HASHLOG_L; ctx->geom.hashLogS = (ctx->geom.flags & B2Z_FLAG_FIND_FAST) ? B2Z_DEF_HASHLOG_L : B2Z_DEF_HASHLOG_S;
                            return 0;
    case B200Z_P_ZSTD_PARSE: if (v < 0 || v > 1) return fail(ctx, B200Z_E_PARAM, "zstd parse mode out of range%s");
                            ctx->geom.flags = (ctx->geom.flags & ~B2Z_FLAG_ZSTD_OPT) | (v ? B2Z_FLAG_ZSTD_OPT : 0u); return 0;
    case B200Z_P_FRAMELOG:  if (v < 17 || v > B2Z_MAX_FRAMELOG) return fail(ctx, B200Z_E_PARAM, "frameLog out of range%s");
                            ctx->geom.frameLog = (uint32_t)v; if (ctx->geom.windowLog > v) ctx->geom.windowLog = (uint32_t)v;
                            ctx->geom.regionLog = v > B2Z_DEF_PLAIN_REGIONLOG ? B2Z_DEF_PLAIN_REGIONLOG : 0u; ctx->geom.ldmLog = 0; return 0;   // (leaves the long mode)
    // long mode: window 2^v bytes, frames of 8 windows (at most 1 GiB) cut into regions of 1 MiB for stage F, + stage L.
    // 0 leaves it (frames of 1 MiB again).
    case B200Z_P_LONG:      if (v != 0 && (v < 21 || v > B2Z_MAX_LONGLOG)) return fail(ctx, B200Z_E_PARAM, "long: window log out of range%s");
                            if (v == 0) { if (ctx->geom.ldmLog) { ctx->geom.frameLog = ctx->geom.windowLog = B2Z_DEF_FRAMELOG; ctx->geom.regionLog = B2Z_DEF_PLAIN_REGIONLOG; } ctx->geom.ldmLog = 0; return 0; }
                            ctx->geom.windowLog = (uint32_t)v; ctx->geom.frameLog = B2Z_LONG_FRAMELOG((uint32_t)v);
                            ctx->geom.regionLog = B2Z_DEF_REGIONLOG; ctx->geom.ldmLog = B2Z_LDM_LOG((uint32_t)v);
                            return 0;
    // both tables live in the shared memory of one SM: 2^L + 2^S entries <= 192 KiB
    case B200Z_P_HASHLOG_L: if (v < 8 || v > 15 || (1u << v) + (1u << ctx->geom.hashLogS) > B2Z_MAX_HASHLOG_SUM_WORDS) return fail(ctx, B200Z_E_PARAM, "hashLogL out of range%s"); ctx->geom.hashLogL = (uint32_t)v; return 0;
    case B200Z_P_HASHLOG_S: if (v < 8 || v > 15 || (1u << v) + (1u << ctx->geom.hashLogL) > B2Z_MAX_HASHLOG_SUM_WORDS) return fail(ctx, B200Z_E_PARAM, "hashLogS out of range%s"); ctx->geom.hashLogS = (uint32_t)v; return 0;
    case B200Z_P_WINDOWLOG: if (v < 10 || v > B2Z_MAX_FRAMELOG) return fail(ctx, B200Z_E_PARAM, "windowLog out of range%s"); ctx->geom.windowLog = (uint32_t)v; return 0;
    case B200Z_P_FLAGS:     if (v & ~3ll) return fail(ctx, B200Z_E_PARAM, "unknown flag bits%s"); ctx->geom.flags = (ctx->geom.flags & ~3u) | (uint32_t)v; return 0;
    case B200Z_P_LZMA2_SLICELOG: if (v < 0 || v > 3) return fail(ctx, B200Z_E_PARAM, "lzma2 sliceLog out of range%s");
                            ctx->geom.flags = (ctx->geom.flags & ~0x700u) | ((uint32_t)v << 8); return 0;
    case B200Z_P_LZMA2_PARSE: if (v < 0 || v > 1) return fail(ctx, B200Z_E_PARAM, "lzma2 parse mode out of range%s");
                            ctx->geom.flags = (ctx->geom.flags & ~B2Z_FLAG_LZ2_OPT) | (v ? B2Z_FLAG_LZ2_OPT : 0u); return 0;
    case B200Z_P_BATCH_LOG: if (v < 22 || v > 36) return fail(ctx, B200Z_E_PARAM, "batchLog out of range%s"); ctx->batchLog = (uint32_t)v; return 0;
    case B200Z_P_REGIONLOG: if (v != 0 && (v < 17 || v > (int64_t)ctx->geom.frameLog)) return fail(ctx, B200Z_E_PARAM, "regionLog out of range%s");
                            ctx->geom.regionLog = (uint32_t)v; return 0;
    case B200Z_P_CHUNKLOG:  if (v < 5 || v > 8) return fail(ctx, B200Z_E_PARAM, "chunkLog out of range%s"); ctx->geom.chunkLog = (uint32_t)v; return 0;
    case B200Z_P_LZMA2_MODEL: if (v < 0 || v > 3) return fail(ctx, B200Z_E_PARAM, "lzma2 model placement out of range%s"); ctx->lz2Mode = (int)v; return 0;
    // each alone here; lc + lp <= 4 is checked when a compression starts (lz2_check_props), as the values arrive one at a time
    case B200Z_P_LZMA2_LC: if (v < 0 || v > 4) return fail(ctx, B200Z_E_PARAM, "lzma2 lc out of range (0..4)%s"); ctx->lz2Lc = (uint32_t)v; return 0;
    case B200Z_P_LZMA2_LP: if (v < 0 || v > 4) return fail(ctx, B200Z_E_PARAM, "lzma2 lp out of range (0..4)%s"); ctx->lz2Lp = (uint32_t)v; return 0;
    case B200Z_P_LZMA2_PB: if (v < 0 || v > 4) return fail(ctx, B200Z_E_PARAM, "lzma2 pb out of range (0..4)%s"); ctx->lz2Pb = (uint32_t)v; return 0;
    case B200Z_P_DEC_JUMP_SEGLOG: if (v < 16 || v > B2Z_DEC_JUMP_SEGLOG) return fail(ctx, B200Z_E_PARAM, "decoder jump segment log out of range%s"); ctx->decJumpSegLog = (uint32_t)v; return 0;
    case B200Z_P_DEC_JUMP: if (v < 0 || v > 2) return fail(ctx, B200Z_E_PARAM, "decoder jump mode out of range%s"); ctx->decJump = (int)v; return 0;
    case B200Z_P_HOST_BATCH_LOG: if (v < 22 || v > 36) return fail(ctx, B200Z_E_PARAM, "hostBatchLog out of range%s"); ctx->hostBatchLog = (uint32_t)v; return 0;
    }
    return fail(ctx, B200Z_E_PARAM, "unknown parameter%s");
}

int b200z_get_param(b200z_ctx* ctx, int param, int64_t* v) {
    if (!ctx || !v) return B200Z_E_PARAM;
    switch (param) {
    case B200Z_P_LEVEL: *v = ctx->level; return 0;
    case B200Z_P_FRAMELOG: *v = ctx->geom.frameLog; return 0;
    case B200Z_P_HASHLOG_L: *v = ctx->geom.hashLogL; return 0;
    case B200Z_P_HASHLOG_S: *v = ctx->geom.hashLogS; return 0;
    case B200Z_P_WINDOWLOG: *v = ctx->geom.windowLog; return 0;
    case B200Z_P_FLAGS: *v = ctx->geom.flags & 3u; return 0;
    case B200Z_P_LZMA2_SLICELOG: *v = B2Z_LZ2_SLICELOG(ctx->geom.flags); return 0;
    case B200Z_P_LZMA2_PARSE: *v = (ctx->geom.flags & B2Z_FLAG_LZ2_OPT) ? 1 : 0; return 0;
    case B200Z_P_ZSTD_PARSE: *v = (ctx->geom.flags & B2Z_FLAG_ZSTD_OPT) ? 1 : 0; return 0;
    case B200Z_P_BATCH_LOG: *v = ctx->batchLog; return 0;
    case B200Z_P_HOST_BATCH_LOG: *v = ctx->hostBatchLog; return 0;
    case B200Z_P_DEC_JUMP: *v = ctx->decJump; return 0;
    case B200Z_P_DEC_JUMP_SEGLOG: *v = ctx->decJumpSegLog; return 0;
    case B200Z_P_LZMA2_MODEL: *v = ctx->lz2Mode; return 0;
    case B200Z_P_LZMA2_LC: *v = ctx->lz2Lc; return 0;
    case B200Z_P_LZMA2_LP: *v = ctx->lz2Lp; return 0;
    case B200Z_P_LZMA2_PB: *v = ctx->lz2Pb; return 0;
    case B200Z_P_CHUNKLOG: *v = ctx->geom.chunkLog; return 0;
    case B200Z_P_LONG: *v = ctx->geom.ldmLog ? ctx->geom.windowLog : 0; return 0;
    case B200Z_P_REGIONLOG: *v = ctx->geom.regionLog; return 0;
    }
    return B200Z_E_PARAM;
}

const char* b200z_last_error(b200z_ctx* ctx) { return ctx ? ctx->err : "no context"; }
double b200z_get_stat(b200z_ctx* ctx, int s) {
    if (!ctx || s <= 0 || s >= 16) return 0.0;
    double v = ctx->stat[s];
    for (b200z_ctx* p : ctx->peers) v += p->stat[s];                // a group reports the sum over its devices
    return v;
}
void b200z_reset_stats(b200z_ctx* ctx) { if (!ctx) return; memset(ctx->stat, 0, sizeof(ctx->stat)); for (b200z_ctx* p : ctx->peers) memset(p->stat, 0, sizeof(p->stat)); }

size_t b200z_zstd_compress_bound(b200z_ctx* ctx, size_t n) {
    const uint32_t fl = ctx ? ctx->geom.frameLog : B2Z_DEF_FRAMELOG;
    const size_t frames = (n >> fl) + 1, blocks = (n >> 17) + frames;
    return n + blocks * 3 + frames * (B2Z_FRAME_HDR_MAX + 12 + 4) + 64;
}

}  // extern "C"

// ---------------------------------------------------------------- encoder driver
// stage F: one CTA per frame, one CTA per SM (its tables fill the SM's shared memory); CTAs loop over frames
static uint32_t find_ctas(const b200z_ctx* ctx, uint64_t nFrames) {
    return (uint32_t)(nFrames < ctx->smCount ? nFrames : ctx->smCount);
}

// does this batch parse by price (stage C + stage P / stage Z) instead of the greedy stage M?  (the per-file batch mode, which
// sets frameSizes, always runs stage M)
static bool price_parse(const EncGeom& g, int codec) {
    return codec == 1 ? (g.flags & B2Z_FLAG_LZ2_OPT) != 0 : ((g.flags & B2Z_FLAG_ZSTD_OPT) != 0 && !g.frameSizes && !g.ldmLog);
}
// the long mode of the Zstandard encoder: frames of many regions (stage F's unit) + stage L.  Per-file batches and method 21 have none.
static bool long_mode(const EncGeom& g, int codec) { return codec == 0 && !g.frameSizes && g.regionLog && g.regionLog < g.frameLog; }
static bool ldm_on(const EncGeom& g, int codec) { return long_mode(g, codec) && g.ldmLog; }

// stage C of the price-based parses: every resident frame-warp owns 7-30 MB of tables
static uint32_t cand_warps(const b200z_ctx* ctx, uint64_t nFrames) {
    const uint64_t cap = (uint64_t)ctx->smCount * 8u;
    return (uint32_t)(nFrames < cap ? nFrames : cap);
}

// LZMA2 encoder context bits -> the flags bits the kernels read (b2z_params.h): none for the defaults, which keep the compile-time
// instantiations
static uint32_t lz2_props_flags(const b200z_ctx* ctx) {
    const uint32_t props = (ctx->lz2Pb * 5u + ctx->lz2Lp) * 9u + ctx->lz2Lc;
    return props == B2Z_LZ2_PROPS ? 0u : (B2Z_FLAG_LZ2_PROPS | (props << 16));
}
int lz2_check_props(b200z_ctx* ctx) {
    if (ctx->lz2Lc + ctx->lz2Lp > 4u) return fail(ctx, B200Z_E_PARAM, "lzma2: lc + lp must not exceed 4%s");
    if (ctx->lz2Mode == 3 && ctx->lz2Lc + ctx->lz2Lp > 3u)
        return fail(ctx, B200Z_E_PARAM, "lzma2: model placement 3 codes lc + lp <= 3 only (its decision queue holds 13-bit probability indices)%s");
    return 0;
}

static int enc_reserve(b200z_ctx* ctx, uint64_t batchBytes, int codec = 0) {
    const uint64_t F = 1ull << ctx->geom.frameLog;
    const uint64_t nFrames = (batchBytes + F - 1) / F;
    const uint64_t nBlocks = (batchBytes + B2Z_BLOCK - 1) / B2Z_BLOCK + 1;
    int bad = 0;
    if (price_parse(ctx->geom, codec)) {                                // price-based parse: stage C's tables and candidate words
        bad |= ctx->tables.reserve(lzma2_cand_table_bytes(ctx->geom, cand_warps(ctx, nFrames)));
        bad |= ctx->cand.reserve((size_t)nFrames * F * LZP_NCAND * 4u);
    } else {                                                            // stage F -> stage G: a candidate word and a choice byte per input byte
        bad |= ctx->cand.reserve((size_t)(nFrames * F + 16) * 4u);
        bad |= ctx->choice.reserve((size_t)(nFrames * F + 16));
        if (ldm_on(ctx->geom, codec)) bad |= ctx->tables.reserve(zstd_enc_ldm_table_words(ctx->geom, nFrames * F) * 4u);
    }
    bad |= ctx->seqs.reserve(nBlocks * B2Z_MAXSEQ * 8ull);
    bad |= ctx->nseq.reserve(nBlocks * 4);
    bad |= ctx->lits.reserve(nBlocks * (size_t)B2Z_BLOCK);
    bad |= ctx->nlit.reserve(nBlocks * 4);
    bad |= ctx->slots.reserve(codec == 1 ? nFrames * lzma2_enc_slices_per_frame(ctx->geom) * lzma2_enc_slot_stride(ctx->geom) : nBlocks * (size_t)B2Z_SLOT);
    bad |= ctx->slotSize.reserve(nBlocks * 4);
    bad |= ctx->blockOff.reserve((nBlocks + 1) * 8);
    bad |= ctx->frameOff.reserve((nFrames * (codec == 1 ? lzma2_enc_slices_per_frame(ctx->geom) : 1u) + 2) * 8);
    bad |= ctx->scalars.reserve(128);                                   // [0] u64 produced bytes, [16] u32 LZMA2 slot overflow, [64] u32 stage F arrival-flag timeout
    bad |= ctx->cks.reserve((nFrames + 2) * 4);
    return bad ? fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s") : 0;
}

// compress [d_src, d_src+n) (n > 0, one batch) to d_dst; returns produced bytes through *produced
static int enc_batch(b200z_ctx* ctx, const uint8_t* d_src, uint64_t n, uint8_t* d_dst, uint64_t* produced, bool stageMOnly,
                     const uint32_t* ready = nullptr, uint32_t readyShift = 0, int codec = 0) {
    int rc = enc_reserve(ctx, n, codec);
    if (rc) return rc;
    EncGeom g = ctx->geom;
    if (codec == 1) g.flags |= lz2_props_flags(ctx);
    const uint64_t F = 1ull << g.frameLog;
    const uint64_t nFrames = (n + F - 1) / F;
    const uint32_t nBlocks = (uint32_t)((n >> 17) + ((n & (B2Z_BLOCK - 1)) ? 1 : 0));
    // blocks are numbered per frame with a fixed stride (frames are multiples of 128 KiB)
    cudaStream_t st = ctx->stream;
    uint32_t* const errFlag = (uint32_t*)ctx->scalars.p + 16;
    auto addMs = [&](int s, int from, int to) { float ms = 0; cudaEventElapsedTime(&ms, ctx->ev[from], ctx->ev[to]); ctx->stat[s] += ms; };
    CU(cudaMemsetAsync(ctx->scalars.p, 0, 128, st));
    CU(cudaEventRecord(ctx->ev[0], st));
    if (price_parse(g, codec)) {
        // price-based parse: stage C (candidates) + stage P (method 21) / stage Z (zstd) instead of the greedy stage M
        if (ready) { CU(cudaEventRecord(ctx->pe[1], ctx->stream2)); CU(cudaStreamWaitEvent(st, ctx->pe[1], 0)); }   // the whole upload first
        launch_lzma2_cand(d_src, n, g, (uint32_t*)ctx->tables.p, cand_warps(ctx, nFrames), (uint32_t*)ctx->cand.p, st);
        CU(cudaGetLastError());
        CU(cudaEventRecord(ctx->ev[4], st));
        if (codec == 1) CU(launch_lzma2_parse(d_src, n, g, (const uint32_t*)ctx->cand.p, (uint64_t*)ctx->seqs.p, (uint32_t*)ctx->nseq.p, st));
        else CU(launch_zstd_enc_parse(d_src, n, g, (const uint32_t*)ctx->cand.p, (uint64_t*)ctx->seqs.p, (uint32_t*)ctx->nseq.p,
                                      (uint8_t*)ctx->lits.p, (uint32_t*)ctx->nlit.p, st));
        CU(cudaEventRecord(ctx->ev[1], st));
        ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 2;
    } else {
        EncGeom gF = g;                                                 // stage F's unit: the frame, or the region of a long frame
        if (long_mode(g, codec)) gF.frameLog = g.regionLog;
        CU(launch_zstd_enc_find(d_src, n, gF, (uint32_t*)ctx->cand.p, find_ctas(ctx, (n + (1ull << gF.frameLog) - 1) >> gF.frameLog), ready, readyShift, errFlag, st));
        if (ldm_on(g, codec)) {
            CU(launch_zstd_enc_ldm(d_src, n, g, (uint32_t*)ctx->cand.p, (uint32_t*)ctx->tables.p, ctx->smCount, st));
            ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 2;
        }
        CU(cudaEventRecord(ctx->ev[4], st));
        CU(launch_zstd_enc_dp(d_src, n, g, (const uint32_t*)ctx->cand.p, (uint8_t*)ctx->choice.p, (uint64_t*)ctx->seqs.p, (uint32_t*)ctx->nseq.p,
                              (uint8_t*)ctx->lits.p, (uint32_t*)ctx->nlit.p, st));
        CU(cudaEventRecord(ctx->ev[1], st));
        ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 2;
    }
    if (stageMOnly) {
        CU(cudaStreamSynchronize(st));
        addMs(B200Z_S_ENC_MATCH_MS, 0, 4); addMs(B200Z_S_ENC_PARSE_MS, 4, 1);
        return 0;
    }
    if (codec == 1) {
        // LZMA2: stage R (range coding, one thread per frame) + assembly of the frame slots into one chunk stream
        const uint32_t LITN = b2z_lz2_litn(b2z_lz2_props(g.flags));
        uint16_t* spill = nullptr;
        const uint64_t nChains = nFrames * lzma2_enc_slices_per_frame(g);
        // auto placement: a global literal model is worth allocating above 11 chains per SM, or wherever the shared-memory slots end first
        const uint32_t spillPerSm = lzma2_enc_smem_chains_per_sm(g.flags) < 11u ? lzma2_enc_smem_chains_per_sm(g.flags) : 11u;
        if (ctx->lz2Mode == 3) {                                    // 32 chains per warp: every chain's whole model in global memory
            if (ctx->decScratch[5].reserve(lzma2_enc_model_bytes((uint32_t)nChains, g.flags))) return fail(ctx, B200Z_E_MEMORY, "LZMA2: model allocation failed%s");
            spill = (uint16_t*)ctx->decScratch[5].p;
        } else
        if (ctx->lz2Mode != 1 && nChains > (uint64_t)spillPerSm * ctx->smCount && ctx->decScratch[5].reserve((size_t)nChains * LITN * 2u) == 0) spill = (uint16_t*)ctx->decScratch[5].p;
        if (ctx->lz2Mode == 2 && !spill) {
            if (ctx->decScratch[5].reserve((size_t)nChains * LITN * 2u)) return fail(ctx, B200Z_E_MEMORY, "LZMA2: model allocation failed%s");
            spill = (uint16_t*)ctx->decScratch[5].p;
        }
        CU(launch_lzma2_enc_range(d_src, n, g, (const uint64_t*)ctx->seqs.p, (const uint32_t*)ctx->nseq.p, (uint8_t*)ctx->slots.p,
                                  (uint32_t*)ctx->slotSize.p, (uint32_t)nFrames, spill, ctx->smCount, ctx->lz2Mode, (uint32_t*)ctx->scalars.p + 4, st));
        CU(cudaEventRecord(ctx->ev[2], st));
        launch_lzma2_enc_assemble((const uint8_t*)ctx->slots.p, (const uint32_t*)ctx->slotSize.p, (uint32_t)nChains, (uint32_t)lzma2_enc_slot_stride(g),
                                  (uint64_t*)ctx->frameOff.p, d_dst, (uint64_t*)ctx->scalars.p, st);
    } else {
        // stage E's records and state words go to the candidate words, which no stage reads after the parse
        launch_zstd_enc_entropy(d_src, n, g, (const uint64_t*)ctx->seqs.p, (const uint32_t*)ctx->nseq.p, (const uint8_t*)ctx->lits.p,
                                (const uint32_t*)ctx->nlit.p, (uint8_t*)ctx->slots.p, (uint32_t*)ctx->slotSize.p, (uint8_t*)ctx->cand.p,
                                nBlocks, ctx->smCount, st);
        CU(cudaGetLastError());
        CU(cudaEventRecord(ctx->ev[2], st));
        launch_zstd_enc_assemble(d_src, n, g, (const uint8_t*)ctx->slots.p, (const uint32_t*)ctx->slotSize.p, nBlocks, (uint64_t*)ctx->blockOff.p,
                                 d_dst, (uint64_t*)ctx->scalars.p, (uint64_t*)ctx->frameOff.p, (uint32_t*)ctx->cks.p, st);
    }
    CU(cudaGetLastError());
    CU(cudaEventRecord(ctx->ev[3], st));
    ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 3;
    uint64_t hs[9] = {0};
    { const int frc = b2z_fetch_small(ctx, hs, ctx->scalars.p, 72, st); if (frc) return frc; }
    if ((uint32_t)hs[8]) return fail(ctx, B200Z_E_CUDA, "upload stalled: an input chunk never arrived%s");
    if (codec == 1 && (uint32_t)hs[2]) return fail(ctx, B200Z_E_CUDA, "LZMA2: frame slot overflow%s");
    *produced = hs[0];
    addMs(B200Z_S_ENC_MATCH_MS, 0, 4); addMs(B200Z_S_ENC_PARSE_MS, 4, 1); addMs(B200Z_S_ENC_ENTROPY_MS, 1, 2); addMs(B200Z_S_ENC_ASSEMBLE_MS, 2, 3);
    return 0;
}

// bytes per batch of a call that codes 2^log at a time: at most 1 GiB for the price-based parses (stage C keeps 16 bytes per input
// byte), at least one frame
static uint64_t batch_bytes(const b200z_ctx* ctx, uint32_t log, int codec) {
    const uint64_t F = 1ull << ctx->geom.frameLog;
    uint64_t batch = 1ull << log;
    if ((ctx->geom.flags & (codec == 1 ? B2Z_FLAG_LZ2_OPT : B2Z_FLAG_ZSTD_OPT)) && batch > (1ull << 30)) batch = 1ull << 30;
    return batch < F ? F : batch;
}

// device-pointer compress of srcSize > 0 bytes: batches of whole frames, one after the other.  LZMA2 (codec 1): the chunks of the next
// batch follow directly, over the end marker of the one before.
static int enc_device_batches(b200z_ctx* ctx, const uint8_t* d_src, uint64_t srcSize, uint8_t* d_dst, int codec, size_t* dstSize) {
    const uint64_t batch = batch_bytes(ctx, ctx->batchLog, codec);
    uint64_t done = 0, outPos = 0;
    while (done < srcSize) {
        const uint64_t n = (srcSize - done) < batch ? (srcSize - done) : batch;
        uint64_t produced = 0;
        const int rc = enc_batch(ctx, d_src + done, n, d_dst + outPos, &produced, false, nullptr, 0, codec);
        if (rc) return rc;
        done += n; outPos += produced;
        if (codec == 1 && done < srcSize) outPos -= 1;
    }
    *dstSize = (size_t)outPos;
    return 0;
}

// Host-pointer upload of n > 0 bytes to d_dst in <= 16 chunks of >= 1 MiB on stream2, each followed by its flag in ctx->ready: the
// kernels start at once and stage F's CTAs wait for their chunk, so the H2D time hides under the match kernel.  *shift: log2 of the
// chunk size, which enc_batch takes.
static int upload_chunked(b200z_ctx* ctx, uint8_t* d_dst, const uint8_t* src, uint64_t n, uint32_t* shift) {
    if (ctx->ready.reserve(256)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
    if (!ctx->hostOne) { if (cudaHostAlloc((void**)&ctx->hostOne, 64, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return fail(ctx, B200Z_E_MEMORY, "pinned allocation failed%s"); } *ctx->hostOne = 1u; }
    uint32_t s = 20; while (((n - 1) >> s) >= 16) s++;
    const uint32_t nChunks = (uint32_t)(((n - 1) >> s) + 1);
    CU(cudaMemsetAsync(ctx->ready.p, 0, 256, ctx->stream));
    CU(cudaEventRecord(ctx->pe[0], ctx->stream));
    CU(cudaStreamWaitEvent(ctx->stream2, ctx->pe[0], 0));
    for (uint32_t c = 0; c < nChunks; c++) {
        const size_t off = (size_t)c << s, len = (n - off) < ((size_t)1 << s) ? (n - off) : ((size_t)1 << s);
        CU(cudaMemcpyAsync(d_dst + off, src + off, len, cudaMemcpyHostToDevice, ctx->stream2));
        CU(cudaMemcpyAsync((uint32_t*)ctx->ready.p + c, ctx->hostOne, 4, cudaMemcpyHostToDevice, ctx->stream2));
    }
    *shift = s;
    return 0;
}

static size_t enc_bound(b200z_ctx* ctx, uint64_t n, int codec) { return codec == 1 ? b200z_lzma2_compress_bound(ctx, n) : b200z_zstd_compress_bound(ctx, n); }

// Host-pointer compress on one device, batch after batch: chunked upload, kernels, download.  srcSize == 0 (zstd only): the empty frame.
static int enc_host_serial(b200z_ctx* ctx, const uint8_t* src, uint64_t srcSize, uint8_t* dst, uint64_t batch, int codec, size_t* dstSize) {
    const uint64_t maxIn = srcSize < batch ? srcSize : batch;
    const size_t bound = enc_bound(ctx, maxIn, codec);
    if (ctx->dIn.reserve(maxIn + 64) || ctx->dOut.reserve(bound)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
    uint8_t* const dIn = (uint8_t*)ctx->dIn.p; uint8_t* const dOut = (uint8_t*)ctx->dOut.p;
    uint64_t done = 0, outPos = 0;
    do {
        const uint64_t n = (srcSize - done) < batch ? (srcSize - done) : batch;
        uint64_t produced = 0;
        if (n == 0) { size_t o = 0; const int rc = b200z_zstd_compress_device(ctx, dIn, 0, dOut, bound, &o); if (rc) return rc; produced = o; }
        else {
            uint32_t shift = 0;
            int rc = upload_chunked(ctx, dIn, src + done, n, &shift);
            if (!rc) rc = enc_batch(ctx, dIn, n, dOut, &produced, false, (const uint32_t*)ctx->ready.p, shift, codec);
            if (rc) { cudaStreamSynchronize(ctx->stream2); return rc; }
        }
        if (codec == 1 && done + n < srcSize) produced -= 1;            // the next batch's chunks follow directly: no end marker in between
        CU(cudaMemcpyAsync(dst + outPos, dOut, produced, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        ctx->stat[B200Z_S_H2D_BYTES] += (double)n; ctx->stat[B200Z_S_D2H_BYTES] += (double)produced;
        done += n; outPos += produced;
    } while (done < srcSize);
    *dstSize = (size_t)outPos;
    return 0;
}

// Host-pointer compress through the batch pipeline (b2z_host_pipeline): batch i of `batch` bytes goes to device i mod N.
static int enc_host_pipelined(b200z_ctx* ctx, const uint8_t* src, uint64_t srcSize, uint8_t* dst, uint64_t batch, int codec, size_t* dstSize) {
    std::vector<HostBatch> batches;
    for (uint64_t off = 0; off < srcSize; off += batch) batches.push_back({ (size_t)off, (size_t)((srcSize - off) < batch ? (srcSize - off) : batch), 0, false });
    const size_t outStride = (enc_bound(ctx, batch, codec) + 255) & ~(size_t)255;
    uint64_t total = 0;
    const int rc = b2z_host_pipeline(ctx, src, dst, batches, batch + 64, outStride, [&](b200z_ctx* c, size_t i, const uint8_t* dIn, uint8_t* dOut, uint64_t* out) {
        const int brc = enc_batch(c, dIn, batches[i].srcLen, dOut, out, false, nullptr, 0, codec);
        if (!brc && codec == 1 && i + 1 < batches.size()) *out -= 1;  // the next batch's chunks follow directly: no end marker in between
        return brc;
    }, &total);
    if (rc) return rc;
    *dstSize = (size_t)total;
    return 0;
}

extern "C" size_t b200z_lzma2_compress_bound(b200z_ctx* ctx, size_t srcSize);
extern "C" uint32_t b200z_crc32_combine(uint32_t crcA, uint32_t crcB, uint64_t lenB);
extern "C" int b200z_zstd_compress_batch_crc_host(b200z_ctx* ctx, const void* src, const uint64_t* sizes, uint32_t nFiles, void* dst, size_t dstCap, uint64_t* dstOffsets, uint32_t* crcs);
static const uint8_t kEmptyFrame[9] = { 0x28, 0xB5, 0x2F, 0xFD, 0x20, 0x00, 0x01, 0x00, 0x00 };

extern "C" {

int b200z_zstd_compress_device(b200z_ctx* ctx, const void* d_src, size_t srcSize, void* d_dst, size_t dstCap, size_t* dstSize) {
    if (!ctx || !dstSize || (!d_src && srcSize) || !d_dst) return B200Z_E_PARAM;
    if ((uintptr_t)d_src & 15u) return fail(ctx, B200Z_E_PARAM, "device source must be 16-byte aligned%s");
    if (dstCap < b200z_zstd_compress_bound(ctx, srcSize)) return fail(ctx, B200Z_E_DSTSIZE, "dstCap < b200z_zstd_compress_bound%s");
    CU(cudaSetDevice(ctx->device));
    if (srcSize == 0) {
        size_t o = 0; uint8_t tmp[32];
        const bool ck = (ctx->geom.flags & 2u) != 0;
        if (ctx->geom.flags & 1u) { const uint8_t k[12] = { 0x50, 0x2A, 0x4D, 0x18, 4, 0, 0, 0, (uint8_t)(ck ? 13 : 9), 0, 0, 0 }; memcpy(tmp, k, 12); o = 12; }
        memcpy(tmp + o, kEmptyFrame, 9); if (ck) tmp[o + 4] = 0x24; o += 9;
        if (ck) { const uint8_t x[4] = { 0x99, 0xE9, 0xD8, 0x51 }; memcpy(tmp + o, x, 4); o += 4; }      // XXH64("") low 32 bits
        CU(cudaMemcpyAsync(d_dst, tmp, o, cudaMemcpyHostToDevice, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        *dstSize = o; return 0;
    }
    return enc_device_batches(ctx, (const uint8_t*)d_src, srcSize, (uint8_t*)d_dst, 0, dstSize);
}

// Host-pointer compress: one batch on one device (and the empty input) takes the chunked upload; several batches and / or several
// devices take the pipeline, H2D copy of batch i+1 | kernels of batch i | D2H copy of batch i-1 on every device.
int b200z_zstd_compress_host(b200z_ctx* ctx, const void* src, size_t srcSize, void* dst, size_t dstCap, size_t* dstSize) {
    if (!ctx || !dstSize || (!src && srcSize) || !dst) return B200Z_E_PARAM;
    if (dstCap < b200z_zstd_compress_bound(ctx, srcSize)) return fail(ctx, B200Z_E_DSTSIZE, "dstCap < b200z_zstd_compress_bound%s");
    CU(cudaSetDevice(ctx->device));
    const uint64_t F = 1ull << ctx->geom.frameLog;
    const uint64_t nDev = 1 + ctx->peers.size();
    uint64_t batch = batch_bytes(ctx, ctx->hostBatchLog, 0);
    if (nDev > 1) {                                              // about four batches per device, none smaller than one frame per SM
        const uint64_t unit = long_mode(ctx->geom, 0) ? 1ull << ctx->geom.regionLog : F;        // what one CTA of stage F takes
        uint64_t per = (srcSize + 4 * nDev - 1) / (4 * nDev), floorB = (uint64_t)ctx->smCount * unit;
        if (per < floorB) per = floorB;
        per = (per + F - 1) / F * F;
        if (per < batch) batch = per;
    }
    {   // whole rounds of stage F's grid (one CTA per SM, one region each): a batch of 1024 regions would end with a partial round (1024 = 7 x 132 + 100 on an H100)
        const uint64_t unit = long_mode(ctx->geom, 0) ? 1ull << ctx->geom.regionLog : F, round = (uint64_t)ctx->smCount * unit;
        if (!(ctx->geom.flags & B2Z_FLAG_ZSTD_OPT) && batch > round && srcSize > batch) { const uint64_t b = batch / round * round; if (b % F == 0) batch = b; }
    }
    if (srcSize == 0 || (nDev == 1 && srcSize <= batch)) return enc_host_serial(ctx, (const uint8_t*)src, srcSize, (uint8_t*)dst, batch, 0, dstSize);
    return enc_host_pipelined(ctx, (const uint8_t*)src, srcSize, (uint8_t*)dst, batch, 0, dstSize);
}

int b200z_zstd_enc_stage_m(b200z_ctx* ctx, const void* d_src, size_t srcSize, uint64_t* seqs, uint32_t* nseq, uint8_t* lits, uint32_t* nlit) {
    if (!ctx || !d_src || !srcSize) return B200Z_E_PARAM;
    CU(cudaSetDevice(ctx->device));
    uint64_t produced = 0;
    int rc = enc_batch(ctx, (const uint8_t*)d_src, srcSize, nullptr, &produced, true);
    if (rc) return rc;
    // per-frame block stride -> dense block numbering of the oracle (identical unless the last frame is short)
    const uint64_t F = 1ull << ctx->geom.frameLog; const uint32_t bpf = (uint32_t)(F >> 17);
    const uint64_t nFrames = (srcSize + F - 1) / F;
    uint64_t dense = 0;
    for (uint64_t f = 0; f < nFrames; f++) {
        const uint64_t fn = (srcSize - f * F) < F ? (srcSize - f * F) : F;
        const uint32_t nb = (uint32_t)((fn + B2Z_BLOCK - 1) / B2Z_BLOCK);
        const size_t sb = (size_t)f * bpf;
        CU(cudaMemcpy(nseq + dense, (uint32_t*)ctx->nseq.p + sb, nb * 4, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(nlit + dense, (uint32_t*)ctx->nlit.p + sb, nb * 4, cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(seqs + dense * B2Z_MAXSEQ, (uint64_t*)ctx->seqs.p + sb * B2Z_MAXSEQ, (size_t)nb * B2Z_MAXSEQ * 8, cudaMemcpyDeviceToHost));
        dense += nb;
    }
    CU(cudaMemcpy(lits, ctx->lits.p, srcSize, cudaMemcpyDeviceToHost));
    return 0;
}

int b200z_zstd_enc_stage_f(b200z_ctx* ctx, const void* d_src, size_t srcSize, uint32_t* cand) {
    if (!ctx || !d_src || !srcSize || !cand) return B200Z_E_PARAM;
    if (price_parse(ctx->geom, 0)) return fail(ctx, B200Z_E_PARAM, "stage F belongs to B200Z_P_ZSTD_PARSE 0%s");
    CU(cudaSetDevice(ctx->device));
    uint64_t produced = 0;
    int rc = enc_batch(ctx, (const uint8_t*)d_src, srcSize, nullptr, &produced, true);
    if (rc) return rc;
    CU(cudaMemcpy(cand, ctx->cand.p, srcSize * 4u, cudaMemcpyDeviceToHost));
    return 0;
}

// ---------------------------------------------------------------- many independent files in one call (BASELINE configs[4])
size_t b200z_zstd_compress_batch_bound(b200z_ctx* ctx, size_t totalBytes, uint32_t nFiles) {
    (void)ctx;
    const size_t frames = (totalBytes >> 17) + nFiles + 1;
    return totalBytes + frames * (3 + B2Z_FRAME_HDR_MAX + 12 + 4) + 64;
}

// src: the files back to back; sizes[i]: bytes of file i.  Every file becomes its own run of 128 KiB frames (first frame of
// file i at dst + dstOffsets[i], dstOffsets[nFiles] = total), so any file can be decoded alone -- the per-file fan-out of a
// non-solid 7z archive (7zUpdate.cpp / 7zEncode.cpp:325-332 run one Code() per file; here one call runs them all).
int b200z_zstd_compress_batch_host(b200z_ctx* ctx, const void* src, const uint64_t* sizes, uint32_t nFiles,
                                   void* dst, size_t dstCap, uint64_t* dstOffsets) {
    return b200z_zstd_compress_batch_crc_host(ctx, src, sizes, nFiles, dst, dstCap, dstOffsets, nullptr);
}

// same, and crcs[i] = CRC32 of file i (7-Zip's CrcCalc: what an archive stores per file), computed from the bytes while they are in HBM:
// 64 KiB pieces on the GPU, folded per file on the host (crc(A||B) = crc(A) x^(8|B|) + crc(B))
int b200z_zstd_compress_batch_crc_host(b200z_ctx* ctx, const void* src, const uint64_t* sizes, uint32_t nFiles,
                                       void* dst, size_t dstCap, uint64_t* dstOffsets, uint32_t* crcs) {
    if (!ctx || !sizes || !dstOffsets || !dst) return B200Z_E_PARAM;
    uint64_t total = 0;
    for (uint32_t i = 0; i < nFiles; i++) total += sizes[i];
    if (total && !src) return B200Z_E_PARAM;
    if (dstCap < b200z_zstd_compress_batch_bound(ctx, (size_t)total, nFiles)) return fail(ctx, B200Z_E_DSTSIZE, "dstCap < b200z_zstd_compress_batch_bound%s");
    CU(cudaSetDevice(ctx->device));
    const EncGeom saved = ctx->geom;
    struct Restore { b200z_ctx* c; EncGeom g; ~Restore() { c->geom = g; } } restore{ctx, saved};
    ctx->geom.frameLog = 17; if (ctx->geom.windowLog > 17) ctx->geom.windowLog = 17;
    const uint64_t F = 1ull << 17;
    uint64_t capFrames = (1ull << ctx->batchLog) >> 17; if (capFrames < 1) capFrames = 1;
    std::vector<uint64_t> off; std::vector<uint32_t> sz, firstFrame;
    uint64_t outPos = 0, srcPos = 0;
    uint32_t file = 0;
    cudaStream_t st = ctx->stream;
    while (file < nFiles) {
        // group whole files into one batch of at most capFrames frames (a single larger file still goes alone)
        off.clear(); sz.clear(); firstFrame.clear();
        const uint32_t file0 = file; const uint64_t src0 = srcPos;
        while (file < nFiles) {
            const uint64_t fr = (sizes[file] + F - 1) / F;
            if (!off.empty() && off.size() + fr > capFrames) break;
            firstFrame.push_back((uint32_t)off.size());
            for (uint64_t k = 0; k < fr; k++) { off.push_back(srcPos - src0 + k * F); sz.push_back((uint32_t)((sizes[file] - k * F) < F ? (sizes[file] - k * F) : F)); }
            srcPos += sizes[file]; file++;
        }
        const uint64_t nFr = off.size(), inBytes = srcPos - src0;
        if (nFr == 0) { for (uint32_t i = file0; i < file; i++) dstOffsets[i] = outPos; continue; }      // only empty files
        const size_t bound = b200z_zstd_compress_bound(ctx, nFr * F);
        if (ctx->dIn.reserve(inBytes + 64) || ctx->batchStage.reserve(nFr * F + 64) || ctx->batchOff.reserve(nFr * 8) || ctx->batchSize.reserve(nFr * 4) ||
            ctx->dOut.reserve(bound)) return fail(ctx, B200Z_E_MEMORY, "device staging allocation failed%s");
        CU(cudaMemcpyAsync(ctx->dIn.p, (const uint8_t*)src + src0, inBytes, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(ctx->batchOff.p, off.data(), nFr * 8, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(ctx->batchSize.p, sz.data(), nFr * 4, cudaMemcpyHostToDevice, st));
        launch_zstd_enc_scatter((const uint8_t*)ctx->dIn.p, (const uint64_t*)ctx->batchOff.p, (const uint32_t*)ctx->batchSize.p, (uint32_t)nFr, 17,
                                (uint8_t*)ctx->batchStage.p, st);
        CU(cudaGetLastError());
        ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
        std::vector<uint32_t> pieceCrc; std::vector<uint64_t> pOff, pLen;
        if (crcs) {                                              // per-file digests from the uploaded bytes: pieces of <= 64 KiB, one GPU thread each
            uint64_t at = 0;
            for (uint32_t i = file0; i < file; i++) { for (uint64_t o = 0; o < sizes[i]; o += 65536) { pOff.push_back(at + o); pLen.push_back(sizes[i] - o < 65536 ? sizes[i] - o : 65536); } at += sizes[i]; }
            const size_t np = pOff.size();
            if (np) {
                if (ctx->crcOff.reserve(np * 8) || ctx->crcLen.reserve(np * 8) || ctx->crcOut.reserve(np * 4)) return fail(ctx, B200Z_E_MEMORY, "device scratch allocation failed%s");
                CU(cudaMemcpyAsync(ctx->crcOff.p, pOff.data(), np * 8, cudaMemcpyHostToDevice, st));
                CU(cudaMemcpyAsync(ctx->crcLen.p, pLen.data(), np * 8, cudaMemcpyHostToDevice, st));
                CU(launch_crc_pieces<uint32_t>((const uint8_t*)ctx->dIn.p, inBytes, 0, (const uint64_t*)ctx->crcOff.p, (const uint64_t*)ctx->crcLen.p, (uint32_t)np, B2Z_CRC32_POLY, (uint32_t*)ctx->crcOut.p, st));
                pieceCrc.resize(np);
                CU(cudaMemcpyAsync(pieceCrc.data(), ctx->crcOut.p, np * 4, cudaMemcpyDeviceToHost, st));
                ctx->stat[B200Z_S_KERNEL_LAUNCHES] += 1;
            }
        }
        ctx->geom.frameSizes = (const uint32_t*)ctx->batchSize.p;
        uint64_t produced = 0;
        int rc = enc_batch(ctx, (const uint8_t*)ctx->batchStage.p, nFr * F, (uint8_t*)ctx->dOut.p, &produced, false);
        ctx->geom.frameSizes = nullptr;
        if (rc) return rc;
        if (outPos + produced > dstCap) return fail(ctx, B200Z_E_DSTSIZE, "destination too small%s");
        std::vector<uint64_t> fo(nFr + 1);
        CU(cudaMemcpyAsync(fo.data(), ctx->frameOff.p, (nFr + 1) * 8, cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync((uint8_t*)dst + outPos, ctx->dOut.p, produced, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        ctx->stat[B200Z_S_H2D_BYTES] += (double)inBytes; ctx->stat[B200Z_S_D2H_BYTES] += (double)produced;
        for (uint32_t i = file0, k = 0; i < file; i++, k++) dstOffsets[i] = outPos + fo[firstFrame[k]];   // an empty file owns no frame: zero length
        if (crcs) {
            size_t pi = 0;
            for (uint32_t i = file0; i < file; i++) {
                uint32_t c = 0;                                  // CRC32 of no bytes
                for (uint64_t o = 0; o < sizes[i]; o += 65536, pi++) c = o ? b200z_crc32_combine(c, pieceCrc[pi], pLen[pi]) : pieceCrc[pi];
                crcs[i] = c;
            }
        }
        outPos += produced;
    }
    dstOffsets[nFiles] = outPos;
    return 0;
}

// ---------------------------------------------------------------- LZMA2 (method 21) encoder
size_t b200z_lzma2_compress_bound(b200z_ctx* ctx, size_t srcSize) {
    const uint32_t fl = ctx ? ctx->geom.frameLog : B2Z_DEF_FRAMELOG;
    const size_t F = (size_t)1 << fl, frames = (srcSize + F - 1) / F;
    return srcSize + frames * ((F / 8192u + 2u) * 8u + 16u) + 64u;      // every finished chunk <= its input + 6, >= 8 KiB of input per chunk
}

int b200z_lzma2_compress_device(b200z_ctx* ctx, const void* d_src, size_t srcSize, void* d_dst, size_t dstCap, size_t* dstSize, uint32_t* dictProp) {
    if (!ctx || !dstSize || (!d_src && srcSize) || !d_dst) return B200Z_E_PARAM;
    { const int prc = lz2_check_props(ctx); if (prc) return prc; }
    if ((uintptr_t)d_src & 15u) return fail(ctx, B200Z_E_PARAM, "device source must be 16-byte aligned%s");
    if (dstCap < b200z_lzma2_compress_bound(ctx, srcSize)) return fail(ctx, B200Z_E_DSTSIZE, "dstCap < b200z_lzma2_compress_bound%s");
    if (dictProp) *dictProp = (ctx->geom.frameLog - 12u) * 2u;           // dictionary = frame size (Lzma2Enc_WriteProperties, Lzma2Enc.c:671)
    CU(cudaSetDevice(ctx->device));
    if (srcSize == 0) {                                                  // the end marker alone
        CU(cudaMemsetAsync(d_dst, 0, 1, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        *dstSize = 1; return 0;
    }
    return enc_device_batches(ctx, (const uint8_t*)d_src, srcSize, (uint8_t*)d_dst, 1, dstSize);
}

// Test tap of the price-based parse: stage C's candidate words and stage P's per-block sequences of a device buffer (one batch)
int b200z_lzma2_enc_stage_cp(b200z_ctx* ctx, const void* d_src, size_t srcSize, uint32_t* cand, uint64_t* seqs, uint32_t* nseq) {
    if (!ctx || (!d_src && srcSize)) return B200Z_E_PARAM;
    if (!(ctx->geom.flags & B2Z_FLAG_LZ2_OPT)) return fail(ctx, B200Z_E_PARAM, "set B200Z_P_LZMA2_PARSE to 1 first%s");
    if (!srcSize) return 0;
    CU(cudaSetDevice(ctx->device));
    uint64_t produced = 0;
    int rc = enc_batch(ctx, (const uint8_t*)d_src, srcSize, nullptr, &produced, true, nullptr, 0, 1);
    if (rc) return rc;
    const uint64_t F = 1ull << ctx->geom.frameLog, nFrames = (srcSize + F - 1) / F;
    const uint64_t nBlocks = (nFrames - 1) * (F >> 17) + ((srcSize - (nFrames - 1) * F + B2Z_BLOCK - 1) / B2Z_BLOCK);   // block-indexed per frame; the last frame may be short
    if (cand) CU(cudaMemcpy(cand, ctx->cand.p, srcSize * LZP_NCAND * 4u, cudaMemcpyDeviceToHost));
    if (seqs) CU(cudaMemcpy(seqs, ctx->seqs.p, nBlocks * B2Z_MAXSEQ * 8ull, cudaMemcpyDeviceToHost));
    if (nseq) CU(cudaMemcpy(nseq, ctx->nseq.p, nBlocks * 4ull, cudaMemcpyDeviceToHost));
    return 0;
}

// Host-pointer form: batches of whole dictionary-reset blocks, dealt over the devices by the pipeline (the role of MtCoder_Code,
// MtCoder.c:445, one level up), or on one device one after the other, each with the chunked upload.
int b200z_lzma2_compress_host(b200z_ctx* ctx, const void* src, size_t srcSize, void* dst, size_t dstCap, size_t* dstSize, uint32_t* dictProp) {
    if (!ctx || !dstSize || (!src && srcSize) || !dst) return B200Z_E_PARAM;
    { const int prc = lz2_check_props(ctx); if (prc) return prc; }
    if (dstCap < b200z_lzma2_compress_bound(ctx, srcSize)) return fail(ctx, B200Z_E_DSTSIZE, "dstCap < b200z_lzma2_compress_bound%s");
    if (dictProp) *dictProp = (ctx->geom.frameLog - 12u) * 2u;
    if (!srcSize) { *(uint8_t*)dst = 0; *dstSize = 1; return 0; }
    CU(cudaSetDevice(ctx->device));
    const uint64_t F = 1ull << ctx->geom.frameLog;
    uint64_t batch = batch_bytes(ctx, ctx->hostBatchLog, 1);
    const uint64_t nDev = 1 + ctx->peers.size();
    if (nDev > 1) {                                              // about four batches per device, none smaller than a frame per SM (or 16 frames for large frames)
        uint64_t per = (srcSize + 4 * nDev - 1) / (4 * nDev), floorB = (F >= (1ull << 23) ? 16ull : (uint64_t)ctx->smCount) * F;
        if (per < floorB) per = floorB;
        per = (per + F - 1) / F * F;
        if (per < batch) batch = per;
    }
    return nDev > 1 && srcSize > batch ? enc_host_pipelined(ctx, (const uint8_t*)src, srcSize, (uint8_t*)dst, batch, 1, dstSize)
                                       : enc_host_serial(ctx, (const uint8_t*)src, srcSize, (uint8_t*)dst, batch, 1, dstSize);
}

// ---------------------------------------------------------------- device memory helpers
int b200z_dev_alloc(b200z_ctx* ctx, void** d_ptr, size_t bytes) {
    if (!ctx || !d_ptr) return B200Z_E_PARAM;
    CU(cudaSetDevice(ctx->device));
    CU(cudaMalloc(d_ptr, bytes ? bytes : 16));
    return 0;
}
int b200z_dev_free(b200z_ctx* ctx, void* d_ptr) { if (!ctx) return B200Z_E_PARAM; CU(cudaSetDevice(ctx->device)); CU(cudaFree(d_ptr)); return 0; }
int b200z_dev_upload(b200z_ctx* ctx, void* d_dst, const void* src, size_t bytes) {
    if (!ctx) return B200Z_E_PARAM;
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(d_dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream));
    ctx->stat[B200Z_S_H2D_BYTES] += (double)bytes; return 0;
}
int b200z_dev_download(b200z_ctx* ctx, void* dst, const void* d_src, size_t bytes) {
    if (!ctx) return B200Z_E_PARAM;
    CU(cudaSetDevice(ctx->device));
    CU(cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream)); CU(cudaStreamSynchronize(ctx->stream));
    ctx->stat[B200Z_S_D2H_BYTES] += (double)bytes; return 0;
}
int b200z_host_alloc_pinned(void** ptr, size_t bytes) {
    if (!ptr) return B200Z_E_PARAM;
    if (cudaHostAlloc(ptr, bytes ? bytes : 16, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return B200Z_E_MEMORY; }
    return 0;
}
int b200z_host_free_pinned(void* ptr) { return cudaFreeHost(ptr) == cudaSuccess ? 0 : B200Z_E_CUDA; }

}  // extern "C"
