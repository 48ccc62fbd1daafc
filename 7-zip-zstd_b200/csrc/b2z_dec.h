// b2z_dec.h -- decoder-side structures and launchers (internal to libb200z.so).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2z {

#define B2Z_DEC_MAXSEQ   65536u      // sequences per block (format max: 128 KiB / 3 < 43691)

// error bits (per block / global)
#define B2Z_DERR_CORRUPT      1u
#define B2Z_DERR_UNSUPPORTED  2u
#define B2Z_DERR_TABLE_FULL   4u
#define B2Z_DERR_DSTSIZE      8u
#define B2Z_DERR_CHECKSUM     16u

struct DecFrame {
    uint64_t srcOff;        // first byte of the frame header
    uint64_t dstOff;        // output offset (filled by the layout kernel)
    uint64_t contentSize;   // ~0 if not declared
    uint64_t windowSize;
    uint64_t regen;         // D0: end offset of the frame in src; from D2 on: sum of block sizes
    uint32_t firstBlock, nBlocks;
    uint32_t checksum;      // 1 if a 4-byte content checksum follows the last block
    uint32_t pad;           // D0: scratch (frame header bytes); from D2 on: index of the frame's first execution unit
    uint64_t endOff;        // offset just past the frame in src (the checksum, if any, is the 4 bytes before it)
    uint32_t jump;          // D2: 1 = the frame's matches are resolved by pointer jumping (stage J) instead of by execution units
    uint32_t nComp;         // D0: compressed blocks of the frame (the only ones that own literal / sequence scratch)
    uint32_t firstSlot;     // D0: scratch slot of the frame's first compressed block
    uint32_t pad4;
};

struct DecBlock {
    uint64_t srcOff;        // first byte of block content (after the 3-byte header)
    uint32_t cSize;         // content bytes (RLE: 1)
    uint32_t rawSize;       // regenerated size for raw/RLE blocks
    uint32_t type;          // 0 raw, 1 RLE, 2 compressed
    uint32_t frame;
    int32_t  hufSrc;        // block whose literals section defines the Huffman table (-1: none needed)
    int32_t  tblSrc[3];     // LL, OF, ML: block whose sequences section defines the table
    uint32_t regen;         // regenerated size            (stage D1)
    uint32_t nbSeq;         // sequences decoded           (stage D1)
    uint32_t litSize;       // literals decoded            (stage D1)
    uint32_t status;        // B2Z_DERR_* bits             (stage D1 / D3)
    // repcode history across the block, symbolically (stage D1): after the block, slot s holds repX[s] if its 2 bits of repSym are 0,
    // else (slot (bits - 1) of the history BEFORE the block) - repX[s].  Lets stage D2 hand every block its starting history
    // without anybody walking the frame's sequences in order.
    uint32_t repX[3], repSym;
    uint32_t repInit[3];    // history at the block's first sequence (stage D2)
    uint32_t nearBehind;    // stage D1: 1 = a match with an explicit offset starts at most one unit's span (512 KiB) before the block's first byte
    uint64_t outRel;        // first output byte of the block, relative to its frame (stage D2)
    uint32_t slot;          // index of the block's 128 KiB literal buffer and 64 Ki-sequence array (compressed blocks, numbered densely; ~0 otherwise)
    uint32_t pad4;
};

#define B2Z_DEC_ROUNDS 4u            // stage D3: 32-byte rounds of a batch's literal / match copies whose loads are issued together
#define B2Z_DEC_RING 4096u           // stage D3: bytes of its own latest output a warp mirrors in shared memory
#define B2Z_DEC_UNIT_BLOCKS 4u       // stage D3: consecutive blocks of a frame executed by one warp (512 KiB of output when the blocks are full)

#define B2Z_DEC_JUMP_MIN_UNITS 8u    // stage J, automatic mode: frames of at least this many units ...
#define B2Z_DEC_JUMP_FINAL 0x80000000u   // stage J: pointer bit "the byte pointed at is final" (a literal of the segment, or any byte before the segment)
#define B2Z_DEC_JUMP_BIAS  0x40000000u   // stage J: pointer = position - segment start + this (sources reach at most a window, <= 2^30 - 16, back)
#define B2Z_DEC_JUMP_SEGLOG 30u          // stage J: the batch's output is resolved in segments of this many bytes, in order
#define B2Z_DEC_JUMP_ROUNDS 32u      // pointer doubling: a chain of n links is resolved after ceil(log2 n) rounds, n < 2^31

struct DecCounts { uint32_t nFrames, nBlocks, status, nUnits; uint64_t srcUsed; uint32_t maxFrameBlocks, nJump, nSlots, pad; };

// stage D0: frame discovery (1 thread; hops over mcmilk size hints when present), then per-frame block indexing
void launch_zstd_dec_find_frames(const uint8_t* src, uint64_t srcSize, DecFrame* frames, uint32_t frameCap, DecCounts* counts, bool useHints, cudaStream_t st);
void launch_zstd_dec_index_blocks(const uint8_t* src, uint64_t srcSize, DecFrame* frames, uint32_t nFrames,
                                  DecBlock* blocks, uint32_t blockCap, DecCounts* counts, cudaStream_t st);
// stage D1: headers, then streams (one thread per stream, decoding tables built in shared memory); literals | sequences on two CUDA streams
void launch_zstd_dec_entropy(const uint8_t* src, uint64_t srcSize, DecBlock* blocks, uint32_t nBlocks,
                             uint8_t* lits, uint64_t* seqs, void* scratch, uint32_t smCount, cudaStream_t st, cudaStream_t stLit, cudaEvent_t evFork, cudaEvent_t evJoin);
size_t zstd_dec_entropy_scratch_bytes(uint32_t nBlocks);
// stage D2: per-frame sizes and output offsets
// jumpMode: 0 = every frame by units (stage D3), 1 = frames whose units form a chain go to stage J, 2 = every frame with a block goes to stage J
void launch_zstd_dec_layout(DecFrame* frames, uint32_t nFrames, DecBlock* blocks, uint64_t dstCap,
                            DecCounts* counts, uint64_t* total, uint32_t jumpMode, cudaStream_t st);
// stage J (frames with DecFrame::jump): literals and one pointer per output byte (J1), pointer doubling (J2), byte gather (J3).
// scratch: zstd_dec_jump_scratch_bytes(total, segLog) -- round flags, one word per output byte of a segment, one byte per 128 of them
size_t zstd_dec_jump_scratch_bytes(uint64_t total, uint32_t segLog /* <= B2Z_DEC_JUMP_SEGLOG */);
void launch_zstd_dec_jump(const uint8_t* src, DecFrame* frames, uint32_t nFrames, DecBlock* blocks, uint32_t nBlocks, const uint8_t* lits, const uint64_t* seqs,
                          uint8_t* dst, uint64_t total, uint32_t segLog, DecCounts* counts, void* scratch, uint32_t smCount, cudaStream_t st);
// stage D3: one warp per unit of B2Z_DEC_UNIT_BLOCKS consecutive blocks of a frame, units taken in order; a match that reaches
// behind its unit waits for the unit that writes those bytes.  unitState: [0] ticket, [1 + u] done flag of unit u -- zeroed here.
size_t zstd_dec_unit_state_bytes(uint32_t nFrames, uint32_t nBlocks);
void launch_zstd_dec_exec(const uint8_t* src, DecFrame* frames, uint32_t nFrames, DecBlock* blocks, uint32_t nBlocks,
                          const uint8_t* lits, const uint64_t* seqs, uint8_t* dst, DecCounts* counts, uint32_t* unitState, uint32_t smCount, cudaStream_t st);

// content checksums (XXH64 low 32 bits) of the frames that carry one: one thread per frame, after D3
void launch_zstd_dec_verify(const uint8_t* src, const DecFrame* frames, uint32_t nFrames, const uint8_t* dst, DecCounts* counts, cudaStream_t st);

}  // namespace b2z
