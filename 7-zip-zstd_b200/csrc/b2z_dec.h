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
    uint32_t pad;           // D0: 1 = the end offset came from a size hint; from D2 on: index of the frame's first execution unit
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

// ---------------------------------------------------------------- frame and block headers (RFC 8878 3.1.1)
// One walk for the D0 prepass (zstd_dec.cu reads through its Src) and the host queries (zstd_dec_api.cu, through HostBytes).  A
// reader has u8 / le24 / le32: little-endian values at a byte offset.
#define B2Z_ZSTD_MAGIC 0xFD2FB528u
#define B2Z_DERR_TRUNCATED 32u       // the walk only: the bytes end inside a frame.  D0 reports it as B2Z_DERR_CORRUPT; a host query
                                     // over a stream read piece by piece waits for more bytes

struct HostBytes {                   // bytes past the end read as 0, as past the end of the device's Src
    const uint8_t* p; uint64_t size;
    __host__ __device__ uint32_t u8(uint64_t off) const { return off < size ? p[off] : 0u; }
    __host__ __device__ uint32_t le24(uint64_t off) const { return u8(off) | u8(off + 1) << 8 | u8(off + 2) << 16; }
    __host__ __device__ uint32_t le32(uint64_t off) const { return le24(off) | u8(off + 3) << 24; }
};

// Whether the frame at ip, whose first 4 bytes are `magic`, is a skippable frame (magic 0x184D2A50 .. 0x184D2A5F); then *size = its
// size with the 8-byte header, which may run past the end (8 when its size field is cut off)
template <class R>
__host__ __device__ inline bool zstd_skippable(const R& r, uint32_t magic, uint64_t ip, uint64_t srcSize, uint64_t* size) {
    if ((magic & 0xFFFFFFF0u) != 0x184D2A50u) return false;
    *size = srcSize - ip < 8 ? 8u : 8u + (uint64_t)r.le32(ip + 4);
    return true;
}

// Block_Maximum_Size = min(Window_Size, 128 KiB) (RFC 8878 3.1.1.2.4)
__host__ __device__ __forceinline__ uint64_t block_max(uint64_t windowSize) { return windowSize < 131072u ? windowSize : 131072u; }

// status: 0, B2Z_DERR_TRUNCATED or B2Z_DERR_CORRUPT (reserved bit, window exponent above 31); the parse stops there.
// unsupported: B2Z_DERR_UNSUPPORTED when a dictionary ID or a window above 1 GiB - 16 was met before that.  The decoder refuses such
// frames, and the dictionary ID outranks a content size field cut short; the host queries describe them all the same.
// blockMax: Block_Maximum_Size from the declared window (windowSize may be cut to the content size).
struct ZstdFrameHdr { uint64_t contentSize, windowSize, blockMax; uint32_t checksum, hdrBytes, fcsBytes, status, unsupported; };

// The frame header at ip, whose magic the caller has checked.  contentSize: ~0 when not declared (fcsBytes = 0).
template <class R>
__host__ __device__ inline ZstdFrameHdr zstd_frame_hdr(const R& r, uint64_t ip, uint64_t srcSize) {
    ZstdFrameHdr h; h.contentSize = ~0ull; h.windowSize = 0; h.blockMax = 0; h.checksum = 0; h.hdrBytes = 0; h.fcsBytes = 0; h.status = 0; h.unsupported = 0;
    if (srcSize - ip < 6) { h.status = B2Z_DERR_TRUNCATED; return h; }
    const uint64_t ip0 = ip;
    const uint32_t fhd = r.u8(ip + 4); ip += 5;
    const uint32_t fcsFlag = fhd >> 6, single = (fhd >> 5) & 1u, didFlag = fhd & 3u;
    h.checksum = (fhd >> 2) & 1u;
    if (fhd & 8u) { h.status = B2Z_DERR_CORRUPT; return h; }
    if (!single) {
        const uint32_t wd = r.u8(ip++); const uint32_t wl = 10u + (wd >> 3);
        if (wl > 31) { h.status = B2Z_DERR_CORRUPT; return h; }
        h.windowSize = (1ull << wl) + ((1ull << wl) >> 3) * (wd & 7u);
    }
    const uint32_t didBytes = didFlag == 3 ? 4u : didFlag;
    uint32_t did = 0; for (uint32_t i = 0; i < didBytes; i++) did |= r.u8(ip + i) << (8 * i);
    ip += didBytes;
    if (did) h.unsupported = B2Z_DERR_UNSUPPORTED;
    h.fcsBytes = fcsFlag == 0 ? single : (fcsFlag == 1 ? 2u : (fcsFlag == 2 ? 4u : 8u));
    if (srcSize < ip || srcSize - ip < h.fcsBytes) { h.status = B2Z_DERR_TRUNCATED; return h; }
    if (h.fcsBytes) { uint64_t fcs = 0; for (uint32_t i = 0; i < h.fcsBytes; i++) fcs |= (uint64_t)r.u8(ip + i) << (8 * i); if (h.fcsBytes == 2) fcs += 256; h.contentSize = fcs; }
    ip += h.fcsBytes;
    if (single) h.windowSize = h.contentSize;
    h.blockMax = block_max(h.windowSize);
    if (!single && h.contentSize != ~0ull && h.contentSize < h.windowSize) h.windowSize = h.contentSize;     // no offset can exceed the content (zstd --long=31 on a small file)
    if (h.windowSize > (1ull << 30) - 16) h.unsupported = B2Z_DERR_UNSUPPORTED;
    h.hdrBytes = (uint32_t)(ip - ip0);
    return h;
}

// The blocks of the frame at `off` whose header h parsed without fault, then its checksum.  emit(index, type, Block_Size field,
// payload offset, payload bytes (RLE: 1)) for every block; a nonzero return stops the walk and becomes its status.  status: 0,
// B2Z_DERR_TRUNCATED, B2Z_DERR_CORRUPT (reserved block type, a block over Block_Maximum_Size) or emit's; end: just past the frame.
struct ZstdBlocks { uint64_t end; uint32_t nBlocks, status; };
template <class R, class Emit>
__host__ __device__ inline ZstdBlocks zstd_walk_blocks(const R& r, uint64_t off, uint64_t srcSize, const ZstdFrameHdr& h, Emit emit) {
    ZstdBlocks w; w.end = 0; w.nBlocks = 0; w.status = 0;
    uint64_t ip = off + h.hdrBytes;
    for (;;) {
        if (srcSize < ip || srcSize - ip < 3) { w.status = B2Z_DERR_TRUNCATED; return w; }
        const uint32_t bh = r.le24(ip); ip += 3;
        const uint32_t last = bh & 1u, type = (bh >> 1) & 3u, bsize = bh >> 3;
        if (type == 3 || bsize > h.blockMax) { w.status = B2Z_DERR_CORRUPT; return w; }
        const uint32_t cSize = type == 1 ? 1u : bsize;
        if (srcSize - ip < cSize) { w.status = B2Z_DERR_TRUNCATED; return w; }
        if ((w.status = emit(w.nBlocks, type, bsize, ip, cSize))) return w;
        w.nBlocks++;
        ip += cSize;
        if (last) break;
    }
    if (h.checksum) { if (srcSize - ip < 4) { w.status = B2Z_DERR_TRUNCATED; return w; } ip += 4; }
    w.end = ip;
    return w;
}
struct ZstdEmitNone { __host__ __device__ uint32_t operator()(uint32_t, uint32_t, uint32_t, uint64_t, uint32_t) const { return 0; } };

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
