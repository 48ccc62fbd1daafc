// b2z_kernels.h -- host-visible launchers of the sm_90a kernels (internal to libb200z.so).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "b2z_params.h"

#define B2Z_DP_WARPS        4       // stage G: warps (= blocks of input) per CTA
#define B2Z_ENT_WARPS       4       // stage E: warps (= blocks of input) per CTA
#define B2Z_SLOT            (B2Z_BODY_CAP + 64u) // per-block output slot: 3-byte header + body (<= B2Z_BODY_CAP), 16-B multiple

namespace b2z {

struct EncGeom {
    uint32_t frameLog, hashLogL, hashLogS, windowLog, flags, chunkLog;
    uint32_t regionLog, ldmLog;      // long mode (B200Z_P_LONG): stage F's unit inside a frame (0 = the frame) and stage L's table log (0 = no stage L)
    const uint32_t* frameSizes;      // null: frames are dense (all 2^frameLog bytes but the last).  Batch mode (frameLog 17, one block
                                     // per frame): bytes of every frame, frames sit at multiples of 2^frameLog in the staging buffer
};
__host__ __device__ inline uint32_t enc_frame_bytes(const EncGeom& g, uint64_t srcSize, uint64_t f) {
    if (g.frameSizes) return g.frameSizes[f];
    const uint64_t F = 1ull << g.frameLog, f0 = f << g.frameLog;
    return (uint32_t)((srcSize - f0) < F ? (srcSize - f0) : F);
}

// stage F (zstd_enc_find.cu): one CTA per frame, both hash tables in shared memory -> one candidate word per position
size_t zstd_enc_find_smem_bytes(const EncGeom& g);
cudaError_t launch_zstd_enc_find(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t* cand /* [srcSize + 16] */, uint32_t nCtas,
                                 const uint32_t* ready /* null, or per-chunk arrival flags */, uint32_t readyShift,
                                 uint32_t* errFlag /* set to 1 when an arrival flag never came */, cudaStream_t st);
// stage L (zstd_enc_ldm.cu), long mode: far matches through per-epoch tables of first occurrences of sampled positions; overwrites candidate words
size_t zstd_enc_ldm_table_words(const EncGeom& g, uint64_t srcSize);
cudaError_t launch_zstd_enc_ldm(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t* cand, uint32_t* tables /* [zstd_enc_ldm_table_words] */, uint32_t smCount, cudaStream_t st);
// stage G (zstd_enc_dp.cu): one warp per 128 KiB block, one lane per 4 KiB segment: minimum-price parse of stage F's candidates
// -> per-block final sequences + literal bytes.  choice: one scratch byte per input byte.
size_t zstd_enc_dp_smem_bytes();
cudaError_t launch_zstd_enc_dp(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint32_t* cand, uint8_t* choice,
                               uint64_t* seqs, uint32_t* nseq, uint8_t* lits, uint32_t* nlit, cudaStream_t st);

// stage Z (zstd_enc_parse.cu): the price-based parse, one warp per 128 KiB block, on stage C's candidate words (lzma2_parse.cu);
// fills the same arrays as stage M.  Dense frames only.
size_t zstd_enc_parse_smem_bytes();
cudaError_t launch_zstd_enc_parse(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint32_t* cand,
                                  uint64_t* seqs, uint32_t* nseq, uint8_t* lits, uint32_t* nlit, cudaStream_t st);

// stage E: E1 (tables and literals, one warp per block), E2 (FSE state chains, 30 per warp), E3 (sequence bitstream, one warp
// per block) -> compressed block (with 3-byte header) in its slot.  scratch: 128 KiB + 3 568 B per block (ENT_SCRATCH_STRIDE),
// which fits in the 4 bytes per input byte of the candidate words, dead once the parse has run.
void launch_zstd_enc_entropy(const uint8_t* src, uint64_t srcSize, const EncGeom& g,
                             const uint64_t* seqs, const uint32_t* nseq, const uint8_t* lits, const uint32_t* nlit,
                             uint8_t* slots, uint32_t* slotSize, uint8_t* scratch, uint32_t nBlocks, uint32_t smCount, cudaStream_t st);

// frame assembly: offsets (one CTA scan) + gather of slots into contiguous frames
void launch_zstd_enc_assemble(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint8_t* slots, const uint32_t* slotSize,
                              uint32_t nBlocks, uint64_t* blockOff /* [nBlocks+1] scratch */, uint8_t* dst,
                              uint64_t* outSize /* device scalar */, uint64_t* frameOff /* [nFrames+1] or null */,
                              uint32_t* cks /* [nFrames] scratch (flag bit1) */, cudaStream_t st);

// batch mode: frame f = size[f] bytes at src + off[f]  ->  stage + (f << frameLog)   (one CTA per frame)
void launch_zstd_enc_scatter(const uint8_t* src, const uint64_t* off, const uint32_t* size, uint32_t nFrames, uint32_t frameLog,
                             uint8_t* stage, cudaStream_t st);

// digests and filters (b2z_crc.cu, b2z_filter.cu): per-piece CRC32 / CRC64 (pieces of 2^pieceLog bytes, or the given ranges), SHA-256 of ranges
template <typename T> cudaError_t launch_crc_pieces(const uint8_t* src, uint64_t n, uint32_t pieceLog, const uint64_t* off, const uint64_t* len,
                                                    uint32_t nPieces, T poly, T* out, cudaStream_t st);
cudaError_t launch_sha256_pieces(const uint8_t* src, const uint64_t* off, const uint64_t* len, uint32_t nPieces, uint32_t* out /* [nPieces][8] */, cudaStream_t st);

}  // namespace b2z
