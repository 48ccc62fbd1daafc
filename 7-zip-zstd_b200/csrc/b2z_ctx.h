// b2z_ctx.h -- the context object behind the C ABI (internal to libb200z.so).
#pragma once
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <new>
#include <vector>
#include "../../include/b200z.h"
#include "b2z_kernels.h"
#include "b2z_dec.h"

struct Arena {                       // grow-only device buffer
    void* p = nullptr; size_t cap = 0;
    int reserve(size_t n) {
        if (n <= cap) return 0;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        if (cudaMalloc(&p, n) != cudaSuccess) { cudaGetLastError(); return -1; }
        cap = n; return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct b200z_ctx {
    int device = 0;
    std::vector<b200z_ctx*> peers;    // multi-device context (b200z_create_multi): the contexts of the other devices; this one is device 0 of the group
    cudaStream_t stream = nullptr;
    cudaStream_t stream2 = nullptr;   // side stream (decoder: literals kernel next to the sequences kernel; host path: uploads)
    cudaStream_t stream3 = nullptr;   // host path: downloads
    cudaEvent_t pe[4] = {};           // host-path pipeline events
    uint32_t hostBatchLog = 30;       // bytes per pipeline batch of the host-pointer entry points: up to 1 GiB, trimmed to whole rounds of stage F's
                                      // one-CTA-per-SM grid (924 frames = 7 rounds on 132 SMs), so H2D | kernels | D2H of consecutive batches overlap.  The decoder
                                      // (one warp per frame in its execute stage) takes batches twice as large
    b2z::EncGeom geom{};
    int level = 3;
    uint32_t batchLog = 31;           // bytes per kernel batch of the device-pointer entry points: 2 GiB keeps the scratch (9.5 bytes per batch byte: candidate
                                      // words 4, choices 1, sequences 2, literals 1, block slots 1.5) near 19 GiB whatever the input size
    uint32_t smCount = 132;           // replaced by the device's count in b200z_create
    uint32_t decJumpSegLog = B2Z_DEC_JUMP_SEGLOG;   // stage J: bytes of output resolved per pass (B200Z_P_DEC_JUMP_SEGLOG; tests use small segments)
    int decJump = 1;                  // Zstandard decoder, stage J (frames resolved by pointer jumping): 0 never, 1 frames whose units form a chain, 2 every frame
    int lz2Mode = 0;                  // LZMA2 decoder literal-model placement: 0 auto, 1 shared memory, 2 global memory
    uint32_t lz2Lc = B2Z_LZ2_LC, lz2Lp = B2Z_LZ2_LP, lz2Pb = B2Z_LZ2_PB;   // LZMA2 encoder context bits (B200Z_P_LZMA2_LC/LP/PB)
    Arena tables, seqs, nseq, lits, nlit, slots, slotSize, blockOff, frameOff, scalars, dIn, dOut, cks, ready, batchStage, batchOff, batchSize, cand, choice, crcOff, crcLen, crcOut;
    uint32_t* hostOne = nullptr;      // pinned constant 1 (chunk-arrival flags of the host-pointer path)
    uint64_t* hostSmall = nullptr;    // 256 pinned bytes the device writes its counters into (b2z_fetch_small)
    Arena decScratch[10];
    cudaEvent_t ev[8] = {};
    double stat[16] = {0};
    char err[256] = {0};
};

static inline int fail(b200z_ctx* c, int code, const char* fmt, const char* detail = "") {
    if (c) snprintf(c->err, sizeof(c->err), fmt, detail);
    return code;
}
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { cudaGetLastError(); \
    return fail(ctx, (e_ == cudaErrorMemoryAllocation) ? B200Z_E_MEMORY : B200Z_E_CUDA, #call ": %s", cudaGetErrorString(e_)); } } while (0)

// Counters back to the host WITHOUT the copy engine: a one-warp kernel stores them into pinned host memory, then the stream is synchronised.
// (A cudaMemcpyAsync of a few bytes queues behind whatever the device-to-host engine is doing -- in the host-pointer pipelines the
// gigabyte download of the previous batch: measured, the kernels of batch k+1 started only when the download of batch k had ended.)
int b2z_fetch_small(b200z_ctx* ctx, void* hostDst, const void* d_src, size_t bytes /* multiple of 8, <= 256 */, cudaStream_t st);

// b2z_host_pipeline.cu: the batch pipeline of the host-pointer entry points, over the devices of ctx (ctx, then its peers).  Batch i
// (srcLen bytes of src at srcOff) goes to worker i mod N, which runs H2D (stream2) | code (stream) | D2H (stream3) over its batches with
// double-buffered staging: 2 x inStride bytes of dIn, 2 x outStride of dOut.  code(c, i, dIn, dOut, &n) codes batch i on c->stream and
// synchronises it; its n output bytes go to dst + the sum of the outputs of batches 0 .. i-1, sizes that are known up front (outKnown)
// or published as the batches are coded.  Returns the first error (a peer's message prefixed with its device), else 0 and *total.
// No copy from src or into dst is pending when it returns, whatever the exit.
struct HostBatch { size_t srcOff, srcLen; uint64_t outSize; bool outKnown; };
using HostCode = std::function<int(b200z_ctx* c, size_t i, const uint8_t* dIn, uint8_t* dOut, uint64_t* out)>;
int b2z_host_pipeline(b200z_ctx* ctx, const uint8_t* src, uint8_t* dst, const std::vector<HostBatch>& batches, size_t inStride, size_t outStride,
                      const HostCode& code, uint64_t* total);

// b2z_filter.cu: b200z_filter_device with units -- unitLog != 0 (encode only): the buffer is a run of independent units of 2^unitLog
// bytes (the xz writer filters every Block on its own)
int b2z_filter_units_device(b200z_ctx* ctx, uint32_t methodId, int encode, void* d_data, size_t n, uint32_t prop, uint32_t unitLog);

// LZMA2 encoder: B200Z_E_PARAM (and last_error) unless lc + lp <= 4 and the model placement codes them; every compression entry checks it first
int lz2_check_props(b200z_ctx* ctx);
