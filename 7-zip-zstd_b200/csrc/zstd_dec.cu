// zstd_dec.cu -- Zstandard decoder kernels (sm_90a), bit-exact for any valid frame whose
// window is <= 2^29 and that needs no dictionary.
//
//   D0 prepass  (1 thread)          walk frame and block headers (sequential by format), record
//                                   per block where its entropy tables come from (treeless
//                                   literals / repeat-mode FSE tables chain back to an earlier block)
//   D1 entropy  (1 warp / block)    Huffman-decode the literals (4 streams -> 4 lanes) and FSE-decode
//                                   the sequences (one backward bitstream -> lane 0) into scratch
//   D2 layout   (1 thread / frame)  block sizes -> frame sizes -> output offsets
//   D3 execute  (1 warp / frame)    literal + match copies, block after block (matches may reach
//                                   into earlier blocks of the frame), repcode history carried
//
// Replaces (reference, /root/reference/C/zstd/): zstd_decompress.c:702,1275,2086 (frame/stream
// loop), zstd_decompress_block.c:63 (block header), :134-340 (literals), huf_decompress.c:385,897,
// entropy_common.c:42,242 (NCount / Huffman stats), zstd_decompress_block.c:485,647,695 (FSE
// tables + sequence header), :1229 (ZSTD_decodeSequence), :1001 (ZSTD_execSequence).
// The sequential statement is oracle/zstd_dec_oracle.c; outputs must be identical.
#include "b2z_device.cuh"
#include "b2z_dec.h"

namespace b2z {

// ---------------------------------------------------------------- format constants
__device__ const uint32_t k_LL_base[36] = { 0,1,2,3,4,5,6,7,8,9,10,11,12,13,14,15,
    16,18,20,22,24,28,32,40,48,64,0x80,0x100,0x200,0x400,0x800,0x1000,0x2000,0x4000,0x8000,0x10000 };
__device__ const uint8_t k_LL_bits[36] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
    1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16 };
__device__ const uint32_t k_ML_base[53] = { 3,4,5,6,7,8,9,10,11,12,13,14,15,16,17,18,
    19,20,21,22,23,24,25,26,27,28,29,30,31,32,33,34,
    35,37,39,41,43,47,51,59,67,83,99,0x83,0x103,0x203,0x403,0x803,0x1003,0x2003,0x4003,0x8003,0x10003 };
__device__ const uint8_t k_ML_bits[53] = { 0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
    0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
    1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16 };
__device__ const int16_t k_LL_defNorm[36] = { 4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,
    2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1 };
__device__ const int16_t k_ML_defNorm[53] = { 1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,
    1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,
    1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1 };
__device__ const int16_t k_OF_defNorm[29] = { 1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,
    1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1 };

// ---------------------------------------------------------------- guarded byte access to the source
struct Src {
    const uint64_t* w; uint64_t nWords; uint64_t size;      // 8-byte aligned buffer, size bytes
    __device__ __forceinline__ uint64_t word(uint64_t i) const { return i < nWords ? __ldg(w + i) : 0ull; }
    __device__ __forceinline__ uint64_t le64(uint64_t off) const {       // unaligned 8 bytes, zero past the end
        const uint64_t i = off >> 3; const uint32_t s = (uint32_t)(off & 7u) * 8u;
        const uint64_t a = word(i), b = s ? word(i + 1) : 0ull;
        return funnel64(a, b, s);
    }
    __device__ __forceinline__ uint32_t u8(uint64_t off) const { return (uint32_t)(word(off >> 3) >> ((off & 7u) * 8u)) & 255u; }
    __device__ __forceinline__ uint32_t le24(uint64_t off) const { return (uint32_t)le64(off) & 0xFFFFFFu; }
    __device__ __forceinline__ uint32_t le32(uint64_t off) const { return (uint32_t)le64(off); }
};

// ---------------------------------------------------------------- literals / sequences header parsing
struct LitHdr { uint32_t type, regen, csize, hdr, streams; bool ok; };
__device__ LitHdr parse_lit_hdr(const Src& S, uint64_t off, uint32_t blockSize) {
    LitHdr h; h.ok = false; h.csize = 0; h.streams = 1; h.regen = 0; h.hdr = 0; h.type = 0;
    if (blockSize < 1) return h;
    const uint64_t v = S.le64(off);
    const uint32_t b0 = (uint32_t)v & 255u;
    h.type = b0 & 3u; const uint32_t sf = (b0 >> 2) & 3u;
    if (h.type <= 1) {
        if (sf == 0 || sf == 2) { h.regen = b0 >> 3; h.hdr = 1; }
        else if (sf == 1) { h.regen = ((uint32_t)v >> 4) & 0xFFFu; h.hdr = 2; }
        else { h.regen = ((uint32_t)v >> 4) & 0xFFFFFu; h.hdr = 3; }
        h.csize = h.type == 0 ? h.regen : 1u;
    } else {
        if (blockSize < 5) return h;
        if (sf <= 1) { h.regen = ((uint32_t)v >> 4) & 0x3FFu; h.csize = ((uint32_t)v >> 14) & 0x3FFu; h.hdr = 3; h.streams = sf == 0 ? 1u : 4u; }
        else if (sf == 2) { h.regen = ((uint32_t)v >> 4) & 0x3FFFu; h.csize = (uint32_t)v >> 18; h.hdr = 4; h.streams = 4; }
        else { h.regen = (uint32_t)(v >> 4) & 0x3FFFFu; h.csize = (uint32_t)(v >> 22) & 0x3FFFFu; h.hdr = 5; h.streams = 4; }
    }
    if (h.regen > 131072u || (uint64_t)h.hdr + h.csize > blockSize) return h;
    h.ok = true; return h;
}

struct SeqHdr { uint32_t nbSeq, modes, hdr; bool ok; };   // hdr = bytes up to and including the modes byte
__device__ SeqHdr parse_seq_hdr(const Src& S, uint64_t off, uint32_t avail) {
    SeqHdr h; h.ok = false; h.nbSeq = 0; h.modes = 0; h.hdr = 0;
    if (avail < 1) return h;
    const uint32_t v = S.le32(off);
    uint32_t n = v & 255u, used = 1;
    if (n >= 128) {
        if (n == 255) { if (avail < 3) return h; n = ((v >> 8) & 0xFFFFu) + 0x7F00u; used = 3; }
        else { if (avail < 2) return h; n = ((n - 128u) << 8) + ((v >> 8) & 255u); used = 2; }
    }
    h.nbSeq = n;
    if (n == 0) { h.hdr = used; h.ok = (used == avail); return h; }
    if (avail < used + 1) return h;
    h.modes = S.u8(off + used); h.hdr = used + 1;
    h.ok = (h.modes & 3u) == 0;
    return h;
}

// ---------------------------------------------------------------- D0: prepass
// Frame discovery is sequential by format (a frame's end is only known by walking its block headers) unless
// the stream carries mcmilk's 12-byte skippable size hints (magic 0x184D2A50, size 4, payload = size of the
// following frame; DOC/Methods-Extern.md:91), which our encoder writes when flag bit0 is set: then one thread
// hops from hint to hint and the per-frame block walks run in parallel (one thread per frame).
//   D0a (1 thread)      frames[f].srcOff / pad (= end offset, 0 if unknown); walks unhinted frames itself
//   D0b (thread/frame)  frame header + block count (and end-offset check)
//   D0c (1 thread)      firstBlock = exclusive scan of the block counts
//   D0d (thread/frame)  block table entries incl. where each block's entropy tables come from
// Block_Maximum_Size = min(Window_Size, 128 KiB) (RFC 8878 3.1.1.2.4)
__device__ __forceinline__ uint64_t block_max(uint64_t windowSize) { return windowSize < 131072u ? windowSize : 131072u; }
struct FrameHdr { uint64_t contentSize, windowSize, blockMax; uint32_t checksum, hdrBytes, status; };     // blockMax: from the declared window
__device__ FrameHdr parse_frame_hdr(const Src& S, uint64_t ip, uint64_t srcSize) {
    FrameHdr h; h.status = 0; h.contentSize = ~0ull; h.windowSize = 0; h.blockMax = 0; h.checksum = 0; h.hdrBytes = 0;
    if (srcSize - ip < 6) { h.status = B2Z_DERR_CORRUPT; return h; }
    const uint64_t ip0 = ip;
    const uint32_t fhd = S.u8(ip + 4); ip += 5;
    const uint32_t fcsFlag = fhd >> 6, single = (fhd >> 5) & 1u, didFlag = fhd & 3u;
    h.checksum = (fhd >> 2) & 1u;
    if (fhd & 8u) { h.status = B2Z_DERR_CORRUPT; return h; }
    if (!single) {
        const uint32_t wd = S.u8(ip++); const uint32_t wl = 10u + (wd >> 3);
        if (wl > 31) { h.status = B2Z_DERR_CORRUPT; return h; }
        h.windowSize = (1ull << wl) + ((1ull << wl) >> 3) * (wd & 7u);
    }
    const uint32_t didBytes = didFlag == 3 ? 4u : didFlag;
    uint32_t did = 0; for (uint32_t i = 0; i < didBytes; i++) did |= S.u8(ip + i) << (8 * i);
    ip += didBytes;
    if (did) { h.status = B2Z_DERR_UNSUPPORTED; return h; }
    const uint32_t fcsBytes = fcsFlag == 0 ? single : (fcsFlag == 1 ? 2u : (fcsFlag == 2 ? 4u : 8u));
    if (srcSize < ip || srcSize - ip < fcsBytes) { h.status = B2Z_DERR_CORRUPT; return h; }
    if (fcsBytes) { uint64_t fcs = 0; for (uint32_t i = 0; i < fcsBytes; i++) fcs |= (uint64_t)S.u8(ip + i) << (8 * i); if (fcsBytes == 2) fcs += 256; h.contentSize = fcs; }
    ip += fcsBytes;
    if (single) h.windowSize = h.contentSize;
    h.blockMax = block_max(h.windowSize);
    if (!single && h.contentSize != ~0ull && h.contentSize < h.windowSize) h.windowSize = h.contentSize;     // no offset can exceed the content (zstd --long=31 on a small file)
    if (h.windowSize > (1ull << 30) - 16) { h.status = B2Z_DERR_UNSUPPORTED; return h; }
    h.hdrBytes = (uint32_t)(ip - ip0);
    return h;
}

// Walk the block headers of one frame starting at `ip` (first block header). Returns the status; *nb = blocks,
// *ipEnd = offset after the last block.  With `out` != null also fills the block entries.
// blockMax: Block_Maximum_Size; no block's size field may exceed it.
__device__ uint32_t walk_blocks(const Src& S, uint64_t ip, uint64_t srcSize, uint64_t blockMax, uint32_t* nbOut, uint64_t* ipEnd,
                                DecBlock* out, uint32_t firstBlock, uint32_t frameIdx, uint32_t blockCap, uint32_t firstSlot = 0, uint32_t* nCompOut = nullptr) {
    uint32_t nb = 0, nComp = 0; int32_t lastHuf = -1, lastTbl[3] = { -1, -1, -1 };
    for (;;) {
        if (srcSize < ip || srcSize - ip < 3) return B2Z_DERR_CORRUPT;
        const uint32_t bh = S.le24(ip); ip += 3;
        const uint32_t last = bh & 1u, type = (bh >> 1) & 3u, bsize = bh >> 3;
        if (type == 3 || bsize > 131072u || bsize > blockMax) return B2Z_DERR_CORRUPT;
        const uint32_t cSize = type == 1 ? 1u : bsize;
        if (srcSize - ip < cSize) return B2Z_DERR_CORRUPT;
        if (out) {
            if (firstBlock + nb >= blockCap) return B2Z_DERR_TABLE_FULL;
            const int32_t self = (int32_t)(firstBlock + nb);
            DecBlock b; b.srcOff = ip; b.type = type; b.frame = frameIdx; b.hufSrc = -1; b.tblSrc[0] = b.tblSrc[1] = b.tblSrc[2] = -1;
            b.regen = 0; b.nbSeq = 0; b.litSize = 0; b.status = 0; b.rawSize = 0; b.cSize = cSize; b.nearBehind = 0;
            b.slot = type == 2 ? firstSlot + nComp : 0xFFFFFFFFu; b.pad4 = 0;              // only compressed blocks own literal / sequence scratch
            if (type != 2) { b.rawSize = bsize; b.regen = bsize; }
            else {
                const LitHdr lh = parse_lit_hdr(S, ip, bsize);
                if (!lh.ok) return B2Z_DERR_CORRUPT;
                if (lh.type == 2) { b.hufSrc = self; lastHuf = self; }
                else if (lh.type == 3) { if (lastHuf < 0) return B2Z_DERR_CORRUPT; b.hufSrc = lastHuf; }
                const uint32_t so = lh.hdr + lh.csize;
                const SeqHdr sh = parse_seq_hdr(S, ip + so, bsize - so);
                if (!sh.ok) return B2Z_DERR_CORRUPT;
                if (sh.nbSeq) {
                    for (int t = 0; t < 3; t++) {
                        const uint32_t mode = (sh.modes >> (6 - 2 * t)) & 3u;      // LL, OF, ML
                        if (mode == 3) { if (lastTbl[t] < 0) return B2Z_DERR_CORRUPT; b.tblSrc[t] = lastTbl[t]; }
                        else { b.tblSrc[t] = self; lastTbl[t] = self; }
                    }
                }
            }
            out[firstBlock + nb] = b;
        }
        nb++; nComp += type == 2;
        ip += cSize;
        if (last) break;
    }
    *nbOut = nb; *ipEnd = ip; if (nCompOut) *nCompOut = nComp;
    return 0;
}

// useHints: trust mcmilk's 12-byte size hints (a skippable frame 0x184D2A50 whose 4-byte payload is the compressed size of the zstd frame
// behind it).  counts->nUnits (unused before stage D2) returns how many were trusted: when the stream then fails to index, the caller
// walks it again without them -- a skippable frame that merely looks like a hint is user data the reference skips (zstd_decompress.c:702).
__global__ void zstd_dec_find_frames_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecFrame* frames, uint32_t frameCap, DecCounts* counts, uint32_t useHints) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t hinted = 0;
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    uint64_t ip = 0; uint32_t nf = 0, status = 0;
    while (ip < srcSize && !status) {
        if (srcSize - ip < 4) { status = B2Z_DERR_CORRUPT; break; }
        const uint32_t magic = S.le32(ip);
        if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {
            if (srcSize - ip < 8) { status = B2Z_DERR_CORRUPT; break; }
            const uint64_t sz = S.le32(ip + 4);
            if (srcSize - ip < 8 + sz) { status = B2Z_DERR_CORRUPT; break; }
            // a size hint? (payload = compressed size of the zstd frame that follows; verified by D0b)
            if (useHints && magic == 0x184D2A50u && sz == 4 && srcSize - ip >= 16 && S.le32(ip + 12) == 0xFD2FB528u) {
                const uint64_t fsz = S.le32(ip + 8);
                if (fsz >= 9 && srcSize - (ip + 12) >= fsz) {
                    if (nf >= frameCap) { status = B2Z_DERR_TABLE_FULL; break; }
                    DecFrame fr; fr.srcOff = ip + 12; fr.dstOff = 0; fr.contentSize = ~0ull; fr.windowSize = 0; fr.regen = ip + 12 + fsz;   // regen: end offset (until D2)
                    fr.firstBlock = 0; fr.nBlocks = 0; fr.checksum = 0; fr.pad = 1; fr.endOff = ip + 12 + fsz; fr.jump = 0; fr.nComp = 0; fr.firstSlot = 0; fr.pad4 = 0;                          // pad: 1 = end offset is a hint
                    frames[nf++] = fr; hinted++;
                    ip += 12 + fsz; continue;
                }
            }
            ip += 8 + sz; continue;
        }
        if (magic != 0xFD2FB528u) { status = B2Z_DERR_CORRUPT; break; }
        if (nf >= frameCap) { status = B2Z_DERR_TABLE_FULL; break; }
        const FrameHdr h = parse_frame_hdr(S, ip, srcSize);
        if (h.status) { status = h.status; break; }
        uint32_t nb; uint64_t end;
        status = walk_blocks(S, ip + h.hdrBytes, srcSize, h.blockMax, &nb, &end, nullptr, 0, nf, 0);
        if (status) break;
        if (h.checksum) { if (srcSize - end < 4) { status = B2Z_DERR_CORRUPT; break; } end += 4; }
        DecFrame fr; fr.srcOff = ip; fr.dstOff = 0; fr.contentSize = ~0ull; fr.windowSize = 0; fr.regen = end; fr.firstBlock = 0; fr.nBlocks = nb; fr.checksum = 0; fr.pad = 0; fr.endOff = end; fr.jump = 0; fr.nComp = 0; fr.firstSlot = 0; fr.pad4 = 0;
        frames[nf++] = fr;
        ip = end;
    }
    counts->nFrames = nf; counts->nBlocks = 0; counts->status = status; counts->srcUsed = ip; counts->nUnits = hinted;
}

__global__ void zstd_dec_count_blocks_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecFrame* frames, uint32_t nFrames, DecCounts* counts) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFrames) return;
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    DecFrame fr = frames[f];
    const FrameHdr h = parse_frame_hdr(S, fr.srcOff, srcSize);
    uint32_t status = h.status, nb = 0, nComp = 0; uint64_t end = 0;
    if (!status) status = walk_blocks(S, fr.srcOff + h.hdrBytes, srcSize, h.blockMax, &nb, &end, nullptr, 0, f, 0, 0, &nComp);
    if (!status && h.checksum) { if (srcSize - end < 4) status = B2Z_DERR_CORRUPT; else end += 4; }
    if (!status && end != fr.regen) status = B2Z_DERR_CORRUPT;          // a size hint that does not match its frame
    fr.contentSize = h.contentSize; fr.windowSize = h.windowSize; fr.checksum = h.checksum; fr.nBlocks = nb; fr.pad = h.hdrBytes; fr.nComp = nComp;
    frames[f] = fr;
    if (status) atomicOr(&counts->status, status);
}

__global__ void zstd_dec_scan_blocks_kernel(DecFrame* frames, uint32_t nFrames, uint32_t blockCap, DecCounts* counts) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t total = 0, most = 0, slots = 0;
    for (uint32_t f = 0; f < nFrames; f++) {
        frames[f].firstBlock = total; total += frames[f].nBlocks; if (frames[f].nBlocks > most) most = frames[f].nBlocks;
        frames[f].firstSlot = slots; slots += frames[f].nComp;
    }
    counts->nBlocks = total; counts->maxFrameBlocks = most; counts->nSlots = slots;
    if (total > blockCap) counts->status |= B2Z_DERR_TABLE_FULL;
}

__global__ void zstd_dec_fill_blocks_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecFrame* frames, uint32_t nFrames,
                                            DecBlock* blocks, uint32_t blockCap, DecCounts* counts) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFrames || counts->status) return;
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    const DecFrame fr = frames[f];
    uint32_t nb; uint64_t end;
    const uint64_t blockMax = parse_frame_hdr(S, fr.srcOff, srcSize).blockMax;           // (fr.windowSize may be cut to the content size)
    const uint32_t status = walk_blocks(S, fr.srcOff + fr.pad, srcSize, blockMax, &nb, &end, blocks, fr.firstBlock, f, blockCap, fr.firstSlot);
    frames[f].regen = 0; frames[f].pad = 0;
    if (status) atomicOr(&counts->status, status);
}

// ---------------------------------------------------------------- bit readers (single lane)
struct FwdBits {                                // LSB-first, used for NCount headers
    const Src* S; uint64_t base; uint32_t size; uint32_t bitpos;
    __device__ __forceinline__ uint32_t peek(uint32_t n) const {
        const uint32_t byte = bitpos >> 3;
        uint64_t v = S->le64(base + byte);
        if (byte + 8 > size) { const uint32_t valid = byte < size ? (size - byte) * 8u : 0u; v = valid ? (v & (valid >= 64 ? ~0ull : ((1ull << valid) - 1ull))) : 0ull; }
        return (uint32_t)(v >> (bitpos & 7u)) & ((1u << n) - 1u);
    }
};

struct BwdBits {                                // backward stream with end mark; bits below the start read as 0
    const Src* S; uint64_t base; int64_t bitpos; int64_t winBit; uint64_t win; bool overflow;
    __device__ __forceinline__ int init(const Src* s, uint64_t b, uint32_t size) {
        S = s; base = b; overflow = false; win = 0; winBit = (int64_t)1 << 40;
        if (!size) return -1;
        const uint32_t lastByte = S->u8(b + size - 1);
        if (!lastByte) return -1;
        bitpos = (int64_t)(size - 1) * 8 + (int64_t)highbit32(lastByte);
        return 0;
    }
    __device__ __forceinline__ void refill(int64_t hi) {            // window = 64 bits ending at byte-rounded hi
        winBit = ((hi + 7) & ~7ll) - 64;
        if (winBit >= 0) win = S->le64(base + (uint64_t)(winBit >> 3));
        else if (winBit > -64) win = S->le64(base) << (uint32_t)(-winBit);
        else win = 0;
    }
    __device__ __forceinline__ uint32_t peek(uint32_t n) {          // n in 1..32, does not consume
        const int64_t lo = bitpos - (int64_t)n;
        if (lo < winBit || bitpos > winBit + 64) refill(bitpos);
        return (uint32_t)(win >> (uint32_t)(lo - winBit)) & (n >= 32 ? 0xFFFFFFFFu : ((1u << n) - 1u));
    }
    __device__ __forceinline__ uint32_t read(uint32_t n) {
        if (!n) return 0;
        const uint32_t v = peek(n);
        bitpos -= n; if (bitpos < 0) overflow = true;
        return v;
    }
};

// ---------------------------------------------------------------- per-warp workspace of D1
struct SeqEnt { uint32_t base; uint8_t nbAdd, nbBits; uint16_t next; };
// ROLE 0 = literals kernel (needs the Huffman table), ROLE 1 = sequences kernel (needs the three FSE tables)
template <int ROLE> struct DecWST {
    uint16_t huf[ROLE == 0 ? 2048 : 64];     // symbol | nbBits << 8
    SeqEnt   tabs[ROLE == 1 ? 1280 : 1];     // LL [0,512), OF [512,768), ML [768,1280)
    __device__ __forceinline__ SeqEnt* tab(int t) { return tabs + (t == 0 ? 0 : (t == 1 ? 512 : 768)); }
    __device__ __forceinline__ const SeqEnt* tab(int t) const { return tabs + (t == 0 ? 0 : (t == 1 ? 512 : 768)); }
    uint32_t tabLog[3];
    uint32_t hufBits;
    int16_t  norm[256];
    uint16_t nxt[256];
    uint8_t  sym[512];           // FSE symbol per state (build scratch) / Huffman weights
};

// FSE normalized counts; returns bytes consumed or 0
__device__ uint32_t fse_read_ncount(int16_t* norm, uint32_t* maxSym, uint32_t* tableLog, const Src& S, uint64_t off, uint32_t size, uint32_t maxLog) {
    if (size < 1) return 0;
    FwdBits b; b.S = &S; b.base = off; b.size = size; b.bitpos = 0;
    const uint32_t al = b.peek(4) + 5u; b.bitpos += 4;
    if (al > maxLog) return 0;
    int32_t remaining = 1 << al;
    uint32_t sym = 0; const uint32_t limit = *maxSym;
    while (remaining > 0 && sym <= limit) {
        const uint32_t nb = highbit32((uint32_t)remaining + 1u) + 1u;
        const uint32_t T = 1u << (nb - 1u), mx = 2u * T - 1u - ((uint32_t)remaining + 1u);
        const uint32_t bits = b.peek(nb);
        uint32_t count;
        if ((bits & (T - 1u)) < mx) { count = bits & (T - 1u); b.bitpos += nb - 1u; }
        else { count = bits & (2u * T - 1u); if (count >= T) count -= mx; b.bitpos += nb; }
        const int32_t proba = (int32_t)count - 1;
        remaining -= proba < 0 ? 1 : proba;
        norm[sym++] = (int16_t)proba;
        if (proba == 0) {
            uint32_t rep;
            do { rep = b.peek(2); b.bitpos += 2; for (uint32_t i = 0; i < rep; i++) { if (sym > limit) return 0; norm[sym++] = 0; } } while (rep == 3);
        }
        if ((b.bitpos >> 3) > size + 1u) return 0;
    }
    if (remaining != 0 || sym == 0) return 0;
    const uint32_t used = (b.bitpos + 7u) >> 3;
    if (used > size) return 0;
    *maxSym = sym - 1u; *tableLog = al;
    return used;
}

// generic FSE decode table: symbol per state in ws->sym, (nbBits, newState) returned through arrays
template <class WS> __device__ bool fse_spread(WS* ws, const int16_t* norm, uint32_t maxSym, uint32_t log) {
    const uint32_t size = 1u << log, mask = size - 1u; uint32_t high = size - 1u;
    for (uint32_t s = 0; s <= maxSym; s++) {
        if (norm[s] == -1) { ws->sym[high--] = (uint8_t)s; ws->nxt[s] = 1; } else ws->nxt[s] = (uint16_t)norm[s];
    }
    const uint32_t step = (size >> 1) + (size >> 3) + 3u; uint32_t pos = 0;
    for (uint32_t s = 0; s <= maxSym; s++)
        for (int i = 0; i < norm[s]; i++) { ws->sym[pos] = (uint8_t)s; pos = (pos + step) & mask; while (pos > high) pos = (pos + step) & mask; }
    return pos == 0;
}

template <class WS> __device__ bool build_seq_table(WS* ws, int t, const int16_t* norm, uint32_t maxSym, uint32_t log) {
    if (!fse_spread(ws, norm, maxSym, log)) return false;
    const uint32_t size = 1u << log;
    for (uint32_t u = 0; u < size; u++) {
        const uint32_t s = ws->sym[u], ns = ws->nxt[s]++;
        SeqEnt e; e.nbBits = (uint8_t)(log - highbit32(ns)); e.next = (uint16_t)((ns << e.nbBits) - size);
        if (t == 0) { e.base = k_LL_base[s]; e.nbAdd = k_LL_bits[s]; }
        else if (t == 2) { e.base = k_ML_base[s]; e.nbAdd = k_ML_bits[s]; }
        else { e.base = 1u << s; e.nbAdd = (uint8_t)s; }
        ws->tab(t)[u] = e;
    }
    ws->tabLog[t] = log;
    return true;
}

// Walk the table descriptions of block `blk`'s sequences section; returns the offset (absolute in src)
// and mode of type t's description.  false on malformed data.
template <class WS> __device__ bool locate_seq_table(const Src& S, const DecBlock& blk, int t, WS* ws, uint64_t* descOff, uint32_t* mode, uint32_t* avail) {
    const LitHdr lh = parse_lit_hdr(S, blk.srcOff, blk.cSize);
    if (!lh.ok) return false;
    const uint32_t so = lh.hdr + lh.csize;
    const SeqHdr sh = parse_seq_hdr(S, blk.srcOff + so, blk.cSize - so);
    if (!sh.ok || !sh.nbSeq) return false;
    uint64_t p = blk.srcOff + so + sh.hdr; uint32_t left = blk.cSize - so - sh.hdr;
    const uint32_t maxSymT[3] = { 35, 31, 52 }, maxLogT[3] = { 9, 8, 9 };
    for (int k = 0; k < 3; k++) {
        const uint32_t m = (sh.modes >> (6 - 2 * k)) & 3u;
        if (k == t) { *descOff = p; *mode = m; *avail = left; return true; }
        uint32_t used = 0;
        if (m == 1) used = 1;
        else if (m == 2) { uint32_t ms = maxSymT[k], lg; used = fse_read_ncount(ws->norm, &ms, &lg, S, p, left, maxLogT[k]); if (!used) return false; }
        if (used > left) return false;
        p += used; left -= used;
    }
    return false;
}

// Huffman decoding table from the description at `off`; returns description bytes or 0
template <class WS> __device__ uint32_t huf_read_table(WS* ws, const Src& S, uint64_t off, uint32_t size) {
    if (size < 1) return 0;
    uint8_t* w = ws->sym; uint32_t nw = 0;
    const uint32_t hb = S.u8(off); uint32_t used;
    if (hb >= 128) {
        nw = hb - 127u; used = 1u + (nw + 1u) / 2u;
        if (used > size) return 0;
        for (uint32_t i = 0; i < nw; i++) { const uint32_t v = S.u8(off + 1 + i / 2); w[i] = (uint8_t)((i & 1u) ? (v & 15u) : (v >> 4)); }
    } else {
        used = 1u + hb;
        if (hb == 0 || used > size) return 0;
        uint32_t maxSym = 255, al;
        const uint32_t hs = fse_read_ncount(ws->norm, &maxSym, &al, S, off + 1, hb, 6);
        if (!hs || hs >= hb) return 0;
        // weights FSE table: symbols in ws->sym[256..], nbBits/newState packed in ws->huf[0..63]
        uint8_t* fsym = ws->sym + 256;
        {
            const uint32_t size2 = 1u << al, mask = size2 - 1u; uint32_t high = size2 - 1u;
            for (uint32_t s = 0; s <= maxSym; s++) { if (ws->norm[s] == -1) { fsym[high--] = (uint8_t)s; ws->nxt[s] = 1; } else ws->nxt[s] = (uint16_t)ws->norm[s]; }
            const uint32_t step = (size2 >> 1) + (size2 >> 3) + 3u; uint32_t pos = 0;
            for (uint32_t s = 0; s <= maxSym; s++)
                for (int i = 0; i < ws->norm[s]; i++) { fsym[pos] = (uint8_t)s; pos = (pos + step) & mask; while (pos > high) pos = (pos + step) & mask; }
            if (pos != 0) return 0;
            for (uint32_t u = 0; u < size2; u++) {
                const uint32_t s = fsym[u], ns = ws->nxt[s]++;
                const uint32_t nbb = al - highbit32(ns);
                ws->huf[u] = (uint16_t)(nbb | ((((ns << nbb) - size2) & 0xFFu) << 8));     // newState < 64
            }
        }
        BwdBits b; if (b.init(&S, off + 1 + hs, hb - hs)) return 0;
        uint32_t s1 = b.read(al), s2 = b.read(al);
        if (b.overflow) return 0;
        for (;;) {
            if (nw > 253) return 0;
            w[nw++] = fsym[s1]; { const uint32_t e = ws->huf[s1]; s1 = (e >> 8) + b.read(e & 255u); }
            if (b.overflow) { w[nw++] = fsym[s2]; break; }
            if (nw > 253) return 0;
            w[nw++] = fsym[s2]; { const uint32_t e = ws->huf[s2]; s2 = (e >> 8) + b.read(e & 255u); }
            if (b.overflow) { w[nw++] = fsym[s1]; break; }
        }
    }
    uint32_t sum = 0, rank[13];
    for (uint32_t r = 0; r < 13; r++) rank[r] = 0;
    for (uint32_t i = 0; i < nw; i++) { if (w[i] > 11) return 0; if (w[i]) sum += 1u << (w[i] - 1u); }
    if (!sum) return 0;
    const uint32_t maxBits = highbit32(sum) + 1u;
    if (maxBits > 11) return 0;
    const uint32_t rest = (1u << maxBits) - sum;
    if (rest & (rest - 1u)) return 0;
    w[nw++] = (uint8_t)(highbit32(rest) + 1u);
    for (uint32_t i = 0; i < nw; i++) rank[w[i]]++;
    if (rank[1] < 2 || (rank[1] & 1u)) return 0;
    uint32_t start[13], pos = 0;
    for (uint32_t r = 1; r <= maxBits; r++) { start[r] = pos; pos += rank[r] << (r - 1u); }
    for (uint32_t s = 0; s < nw; s++) {
        const uint32_t r = w[s]; if (!r) continue;
        const uint32_t len = 1u << (r - 1u); const uint16_t e = (uint16_t)(s | ((maxBits + 1u - r) << 8));
        for (uint32_t i = 0; i < len; i++) ws->huf[start[r] + i] = e;
        start[r] += len;
    }
    ws->hufBits = maxBits;
    return used;
}

// Hot-loop reader (32-bit arithmetic): `cont` holds stream bytes [bytePos, bytePos+8); the next unread bit is
// bit (63 - consumed) of it.  After reload() consumed <= 7, so 57 bits can be read before the next reload.
// Bytes below the stream start read as zero; left() < 0 means the stream was over-read.
struct FastBwd {
    const Src* S; uint64_t base; uint64_t cont; int32_t bytePos; uint32_t consumed;
    __device__ __forceinline__ uint64_t fetch() const {
        if (bytePos >= 0) return S->le64(base + (uint32_t)bytePos);
        if (bytePos > -8) return S->le64(base) << ((uint32_t)(-bytePos) * 8u);
        return 0ull;
    }
    __device__ __forceinline__ int init(const Src* s, uint64_t b, uint32_t size) {
        S = s; base = b;
        if (!size) return -1;
        const uint32_t lastByte = S->u8(b + size - 1);
        if (!lastByte) return -1;
        bytePos = (int32_t)size - 8; consumed = 8u - highbit32(lastByte);      // skip the padding and the end mark
        cont = fetch();
        return 0;
    }
    __device__ __forceinline__ void reload() { bytePos -= (int32_t)(consumed >> 3); consumed &= 7u; cont = fetch(); }
    __device__ __forceinline__ uint32_t read(uint32_t n) {                      // n <= 32 (0 allowed)
        const uint32_t v = (uint32_t)(((cont << consumed) >> 1) >> (63u - n));
        consumed += n;
        return v;
    }
    __device__ __forceinline__ int32_t left() const { return bytePos * 8 + 64 - (int32_t)consumed; }   // unread bits
};

// one Huffman stream, one lane
template <class WS> __device__ bool huf_decode_stream(const WS* ws, const Src& S, uint64_t off, uint32_t size, uint8_t* dst, uint32_t n) {
    FastBwd b; if (b.init(&S, off, size)) return false;
    const uint32_t mb = ws->hufBits;
    for (uint32_t i = 0; i < n; i++) {
        if (b.consumed > 64u - 11u) b.reload();
        const uint32_t e = ws->huf[(uint32_t)((b.cont << b.consumed) >> (64u - mb))];
        dst[i] = (uint8_t)e; b.consumed += (e >> 8);
    }
    return b.left() == 0;
}

// ---------------------------------------------------------------- D1: entropy decode
#define SEQ_PACK(ob, ll, ml) ((uint64_t)(ob) | ((uint64_t)(ll) << 30) | ((uint64_t)((ml) - 3u) << 47))

// Table stage, one warp per compressed block.  ROLE 0: raw/RLE literals are expanded here, for Huffman literals the
// decoding table is built (lane 0) and spilled to global scratch; ROLE 1: the three FSE tables of the sequences
// section are built and spilled.  The serial bitstreams themselves are decoded by the *_streams kernels below with
// ONE THREAD PER STREAM, so that thousands of dependent chains overlap instead of one per warp.
struct LitJob { uint64_t off; uint32_t size, regen, streams, hufBits; };
struct SeqJob { uint64_t bsOff; uint32_t bsLeft, nbSeq, litRegen, logs; };
#define D1_WARPS(ROLE) ((ROLE) == 0 ? 6 : 4)
template <int ROLE> __global__ void __launch_bounds__(D1_WARPS(ROLE) * 32)
zstd_dec_entropy_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecBlock* __restrict__ blocks, uint32_t nBlocks,
                        uint8_t* __restrict__ lits, uint16_t* __restrict__ hufTabs, LitJob* __restrict__ litJobs,
                        SeqEnt* __restrict__ seqTabs, SeqJob* __restrict__ seqJobs) {
    typedef DecWST<ROLE> DecWS;
    __shared__ DecWS wsAll[D1_WARPS(ROLE)];
    const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
    DecWS* ws = &wsAll[wib];
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    for (uint32_t bi = blockIdx.x * D1_WARPS(ROLE) + wib; bi < nBlocks; bi += gridDim.x * D1_WARPS(ROLE)) {
        const DecBlock blk = blocks[bi];
        if (blk.type != 2) continue;
        uint32_t err = 0;
        const LitHdr lh = parse_lit_hdr(S, blk.srcOff, blk.cSize);
        uint8_t* lit = lits + (size_t)blk.slot * 131072u;
        // ---- literals
        if (ROLE == 0) {
        if (lh.type == 0) { for (uint32_t i = lane; i < lh.regen; i += 32) lit[i] = (uint8_t)S.u8(blk.srcOff + lh.hdr + i); }
        else if (lh.type == 1) { const uint8_t v = (uint8_t)S.u8(blk.srcOff + lh.hdr); for (uint32_t i = lane; i < lh.regen; i += 32) lit[i] = v; }
        else {
            uint32_t tdesc = 0;                                  // this block's own table description bytes
            if (lane == 0) {
                const DecBlock sb = blocks[blk.hufSrc];
                const LitHdr sh = parse_lit_hdr(S, sb.srcOff, sb.cSize);
                const uint32_t u = (sh.ok && sh.type == 2) ? huf_read_table(ws, S, sb.srcOff + sh.hdr, sh.csize) : 0u;
                if (!u) err = B2Z_DERR_CORRUPT;
                if (lh.type == 2) tdesc = u;
            }
            err = __shfl_sync(B2Z_FULL, err, 0); tdesc = __shfl_sync(B2Z_FULL, tdesc, 0);
            __syncwarp();
            if (!err) {
                // spill the decoding table; the streams are decoded by zstd_dec_lit_streams_kernel (one thread per stream)
                uint16_t* gt = hufTabs + (size_t)bi * 2048u;
                const uint32_t nEnt = 1u << ws->hufBits;
                for (uint32_t i = lane; i < nEnt; i += 32) gt[i] = ws->huf[i];
                if (lane == 0) { LitJob j; j.off = blk.srcOff + lh.hdr + tdesc; j.size = tdesc <= lh.csize ? lh.csize - tdesc : 0xFFFFFFFFu; j.regen = lh.regen; j.streams = lh.streams; j.hufBits = ws->hufBits; litJobs[bi] = j; }
            }
        }
        if (lane == 0 && (err || lh.type < 2)) { LitJob j; j.off = 0; j.size = 0; j.regen = 0; j.streams = 0; j.hufBits = 0; litJobs[bi] = j; }
        if (lane == 0 && err) atomicOr(&blocks[bi].status, err);
        }
        __syncwarp();
        // ---- sequences (lane 0)
        uint32_t nbSeq = 0;
        if (ROLE == 1) {
        SeqJob job; job.bsOff = 0; job.bsLeft = 0; job.nbSeq = 0; job.litRegen = lh.regen; job.logs = 0;
        if (lane == 0 && !err) {
            const uint32_t so = lh.hdr + lh.csize;
            const SeqHdr sh = parse_seq_hdr(S, blk.srcOff + so, blk.cSize - so);
            nbSeq = sh.nbSeq;
            if (nbSeq > B2Z_DEC_MAXSEQ) err = B2Z_DERR_CORRUPT;
            if (nbSeq && !err) {
                const uint32_t maxSymT[3] = { 35, 31, 52 }, maxLogT[3] = { 9, 8, 9 }, defMax[3] = { 35, 28, 52 }, defLog[3] = { 6, 5, 6 };
                uint64_t bsOff = blk.srcOff + so + sh.hdr; uint32_t bsLeft = blk.cSize - so - sh.hdr;
                for (int t = 0; t < 3 && !err; t++) {
                    uint64_t d; uint32_t mode, avail;
                    const uint32_t ownMode = (sh.modes >> (6 - 2 * t)) & 3u;
                    if (ownMode == 3) {
                        if (!locate_seq_table(S, blocks[blk.tblSrc[t]], t, ws, &d, &mode, &avail) || mode == 3) { err = B2Z_DERR_CORRUPT; break; }
                    } else { d = bsOff; mode = ownMode; avail = bsLeft; }
                    uint32_t used = 0;
                    if (mode == 0) {
                        const int16_t* dn = t == 0 ? k_LL_defNorm : (t == 1 ? k_OF_defNorm : k_ML_defNorm);
                        for (uint32_t s = 0; s <= defMax[t]; s++) ws->norm[s] = dn[s];
                        if (!build_seq_table(ws, t, ws->norm, defMax[t], defLog[t])) err = B2Z_DERR_CORRUPT;
                    } else if (mode == 1) {
                        const uint32_t s = S.u8(d);
                        if (avail < 1 || s > maxSymT[t]) err = B2Z_DERR_CORRUPT;
                        else {
                            SeqEnt e; e.nbBits = 0; e.next = 0;
                            if (t == 0) { e.base = k_LL_base[s]; e.nbAdd = k_LL_bits[s]; } else if (t == 2) { e.base = k_ML_base[s]; e.nbAdd = k_ML_bits[s]; } else { e.base = 1u << s; e.nbAdd = (uint8_t)s; }
                            ws->tab(t)[0] = e; ws->tabLog[t] = 0; used = 1;
                        }
                    } else {
                        uint32_t ms = maxSymT[t], lg;
                        used = fse_read_ncount(ws->norm, &ms, &lg, S, d, avail, maxLogT[t]);
                        if (!used || !build_seq_table(ws, t, ws->norm, ms, lg)) err = B2Z_DERR_CORRUPT;
                    }
                    if (ownMode != 3) { if (used > bsLeft) err = B2Z_DERR_CORRUPT; else { bsOff += used; bsLeft -= used; } }
                }
                if (!err) { job.bsOff = bsOff; job.bsLeft = bsLeft; job.nbSeq = nbSeq; job.litRegen = lh.regen; job.logs = ws->tabLog[0] | (ws->tabLog[1] << 8) | (ws->tabLog[2] << 16); }
            }
        }
        err = __shfl_sync(B2Z_FULL, err, 0); nbSeq = __shfl_sync(B2Z_FULL, nbSeq, 0);
        __syncwarp();                                                 // lane 0's tables are visible to the warp
        if (!err && nbSeq) {                                          // spill the three tables (LL 512 | OF 256 | ML 512 entries)
            uint2* gt = reinterpret_cast<uint2*>(seqTabs + (size_t)bi * 1280u);
            const uint2* st2 = reinterpret_cast<const uint2*>(ws->tabs);
            const uint32_t nL = 1u << ws->tabLog[0], nO = 1u << ws->tabLog[1], nM = 1u << ws->tabLog[2];
            for (uint32_t i = lane; i < nL; i += 32) gt[i] = st2[i];
            for (uint32_t i = lane; i < nO; i += 32) gt[512 + i] = st2[512 + i];
            for (uint32_t i = lane; i < nM; i += 32) gt[768 + i] = st2[768 + i];
        }
        if (lane == 0) {
            if (err) { job.nbSeq = 0; job.bsLeft = 0; }
            if (!nbSeq && !err) { job.bsOff = 0; job.bsLeft = 0; job.nbSeq = 0; job.litRegen = lh.regen; job.logs = 0; }
            seqJobs[bi] = job;
            blocks[bi].regen = (err || nbSeq) ? 0u : lh.regen; blocks[bi].nbSeq = 0; blocks[bi].litSize = lh.regen; if (err) atomicOr(&blocks[bi].status, err);
        }
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------- D1b: one thread per stream
// Literal streams.  The decoding tables (up to 4 KiB per block, 128 MB for the 32 768 blocks of 4 GiB) do not fit L2 while every stream
// of the input is in flight, and a look-up per symbol from HBM was what this kernel waited for.  A CTA therefore
// serves LIT_BLOCKS blocks (4 streams each) and first copies their tables into shared memory: the per-symbol chain is then two shifts,
// one shared-memory load and an add.
#define B2Z_LIT_BLOCKS 16u
__global__ void __launch_bounds__(B2Z_LIT_BLOCKS * 4u)
zstd_dec_lit_streams_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecBlock* __restrict__ blocks, uint32_t nBlocks,
                            uint8_t* __restrict__ lits, const uint16_t* __restrict__ hufTabs, const LitJob* __restrict__ litJobs) {
    B2Z_EXTERN_SMEM(uint16_t, smTab);                                   // [B2Z_LIT_BLOCKS][2048]
    const uint32_t b0 = blockIdx.x * B2Z_LIT_BLOCKS;
    {   // stage the tables of this CTA's blocks (16-byte copies; a block without Huffman streams has none)
        const uint4* g4 = reinterpret_cast<const uint4*>(hufTabs + (size_t)b0 * 2048u);
        uint4* s4 = reinterpret_cast<uint4*>(smTab);
        for (uint32_t i = threadIdx.x; i < B2Z_LIT_BLOCKS * 256u; i += B2Z_LIT_BLOCKS * 4u) {
            const uint32_t bb = b0 + (i >> 8);
            if (bb < nBlocks && blocks[bb].type == 2) {                  // (raw / RLE blocks have no job record: nothing was written there)
                const LitJob jj = litJobs[bb];
                if (jj.streams && (i & 255u) < ((1u << jj.hufBits) + 7u) / 8u) s4[i] = __ldg(g4 + i);
            }
        }
    }
    __syncthreads();
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t bi = t >> 2, k = t & 3u;
    if (bi >= nBlocks) return;
    const LitJob j = litJobs[bi];
    if (!j.streams || blocks[bi].type != 2) return;
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    uint8_t* lit = lits + (size_t)blocks[bi].slot * 131072u;
    const uint16_t* tab = smTab + (size_t)(bi - b0) * 2048u;
    bool ok = true;
    uint64_t off = 0; uint32_t size = 0, cnt = 0; uint8_t* dst = lit;
    if (j.size == 0xFFFFFFFFu) ok = false;
    else if (j.streams == 1) { if (k) return; off = j.off; size = j.size; cnt = j.regen; }
    else {
        if (j.size < 6) ok = false;
        else {
            const uint64_t jt = S.le64(j.off);
            const uint32_t s1 = (uint32_t)jt & 0xFFFFu, s2 = (uint32_t)(jt >> 16) & 0xFFFFu, s3 = (uint32_t)(jt >> 32) & 0xFFFFu;
            const uint32_t seg = (j.regen + 3u) / 4u;
            if (6u + s1 + s2 + s3 > j.size || seg * 3u > j.regen) ok = false;
            else {
                const uint32_t s4 = j.size - 6u - s1 - s2 - s3;
                const uint32_t so = k == 0 ? 0u : (k == 1 ? s1 : (k == 2 ? s1 + s2 : s1 + s2 + s3));
                size = k == 0 ? s1 : (k == 1 ? s2 : (k == 2 ? s3 : s4));
                cnt = k < 3 ? seg : j.regen - 3u * seg;
                off = j.off + 6u + so; dst = lit + k * seg;
            }
        }
    }
    if (ok) {
        FastBwd b;
        if (b.init(&S, off, size)) ok = false;
        else {
            const uint32_t mb = j.hufBits;
            // symbols are gathered eight at a time and stored as one aligned word (head and tail byte by byte): every lane writes its own stream
            uint32_t i = 0;
            const uint32_t head = (uint32_t)((8u - ((uintptr_t)dst & 7u)) & 7u);
            for (; i < cnt && i < head; i++) {
                if (b.consumed > 64u - 11u) b.reload();
                const uint32_t e = tab[(uint32_t)((b.cont << b.consumed) >> (64u - mb))];
                dst[i] = (uint8_t)e; b.consumed += (e >> 8);
            }
            for (; i + 8u <= cnt; i += 8u) {
                uint64_t acc = 0;
#pragma unroll
                for (uint32_t q = 0; q < 8u; q++) {
                    if (b.consumed > 64u - 11u) b.reload();
                    const uint32_t e = tab[(uint32_t)((b.cont << b.consumed) >> (64u - mb))];
                    acc |= (uint64_t)(e & 255u) << (8u * q); b.consumed += (e >> 8);
                }
                *reinterpret_cast<uint64_t*>(dst + i) = acc;
            }
            for (; i < cnt; i++) {
                if (b.consumed > 64u - 11u) b.reload();
                const uint32_t e = tab[(uint32_t)((b.cont << b.consumed) >> (64u - mb))];
                dst[i] = (uint8_t)e; b.consumed += (e >> 8);
            }
            ok = b.left() == 0;
        }
    }
    if (!ok) atomicOr(&blocks[bi].status, B2Z_DERR_CORRUPT);
}

__global__ void __launch_bounds__(128)
zstd_dec_seq_streams_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecBlock* __restrict__ blocks, uint32_t nBlocks,
                            uint64_t* __restrict__ seqs, const SeqEnt* __restrict__ seqTabs, const SeqJob* __restrict__ seqJobs) {
    const uint32_t bi = blockIdx.x * blockDim.x + threadIdx.x;
    if (bi >= nBlocks || blocks[bi].type != 2) return;
    const SeqJob j = seqJobs[bi];
    if (!j.nbSeq) return;
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    const uint2* __restrict__ tab = reinterpret_cast<const uint2*>(seqTabs + (size_t)bi * 1280u);
    uint32_t err = 0, regen = 0;
    FastBwd b;
    if (b.init(&S, j.bsOff, j.bsLeft)) err = B2Z_DERR_CORRUPT;
    else {
        uint32_t sL = b.read(j.logs & 255u), sO = b.read((j.logs >> 8) & 255u), sM = b.read((j.logs >> 16) & 255u);   // <= 26 bits
        if (b.left() < 0) err = B2Z_DERR_CORRUPT;
        uint64_t* out = seqs + (size_t)blocks[bi].slot * B2Z_DEC_MAXSEQ;
        uint32_t litUsed = 0, total = 0, near = 0;
        // the repcode history as a function of the history before the block (b2z_dec.h DecBlock::repX): slot = value (sym 0) or
        // (initial slot sym - 1) minus value.  ZSTD_decodeSequence's update rules, zstd_decompress_block.c:1290-1312
        uint32_t v0 = 0, v1 = 0, v2 = 0, y0 = 1, y1 = 2, y2 = 3;
        for (uint32_t i = 0; i < j.nbSeq && !err; i++) {
            const uint2 rL = __ldg(tab + sL), rO = __ldg(tab + 512u + sO), rM = __ldg(tab + 768u + sM);     // {base, nbAdd | nbBits<<8 | next<<16}
            const uint32_t aL = rL.y & 255u, aO = rO.y & 255u, aM = rM.y & 255u;
            if (aO > 30u) { err = B2Z_DERR_UNSUPPORTED; break; }
            b.reload();
            const uint32_t ob = rO.x + b.read(aO);
            if (aO + aM + aL > 56u) b.reload();
            const uint32_t ml = rM.x + b.read(aM);
            const uint32_t ll = rL.x + b.read(aL);
            if (i + 1 < j.nbSeq) {
                if (aO + aM + aL > 30u) b.reload();                                                     // + <= 26 state bits
                sL = (rL.y >> 16) + b.read((rL.y >> 8) & 255u); sM = (rM.y >> 16) + b.read((rM.y >> 8) & 255u); sO = (rO.y >> 16) + b.read((rO.y >> 8) & 255u);
            }
            litUsed += ll; total += ll + ml;
            if (b.left() < 0 || litUsed > j.litRegen || total > 131072u || ob >= (1u << 30)) { err = B2Z_DERR_CORRUPT; break; }
            out[i] = SEQ_PACK(ob, ll, ml);
            // a source at most one unit's span before the block: the block's unit cannot run beside the unit before it (stage D2 counts these)
            near |= (uint32_t)(ob > 3u && ob - 3u > total - ml && ob - 3u - (total - ml) <= B2Z_DEC_UNIT_BLOCKS * 131072u);
            if (ob > 3u) { v2 = v1; y2 = y1; v1 = v0; y1 = y0; v0 = ob - 3u; y0 = 0u; }
            else {
                const uint32_t idx = ob - 1u + (ll == 0u);
                if (idx == 1u) { const uint32_t tv = v0, ty = y0; v0 = v1; y0 = y1; v1 = tv; y1 = ty; }
                else if (idx == 2u) { const uint32_t tv = v2, ty = y2; v2 = v1; y2 = y1; v1 = v0; y1 = y0; v0 = tv; y0 = ty; }
                else if (idx == 3u) { v2 = v1; y2 = y1; v1 = v0; y1 = y0; v0 = y0 ? v0 + 1u : v0 - 1u; }      // rep0 - 1: one more to subtract, or a smaller value
            }
        }
        blocks[bi].repX[0] = v0; blocks[bi].repX[1] = v1; blocks[bi].repX[2] = v2; blocks[bi].repSym = y0 | (y1 << 2) | (y2 << 4);
        blocks[bi].nearBehind = near;
        if (!err && b.left() != 0) err = B2Z_DERR_CORRUPT;
        regen = total + (j.litRegen - litUsed);
        if (regen > 131072u) err = B2Z_DERR_CORRUPT;
    }
    blocks[bi].regen = err ? 0u : regen; blocks[bi].nbSeq = err ? 0u : j.nbSeq;
    if (err) atomicOr(&blocks[bi].status, err);
}

// ---------------------------------------------------------------- D2: layout
// jumpMode (b2z_dec.h): which frames leave the execution units for stage J.  Automatic: a frame of >= B2Z_DEC_JUMP_MIN_UNITS units in which
// three consecutive units (or three in four of all) start with a block that copies from the unit before it -- a sliding-window frame (what
// the reference's encoder writes: one frame per stream, ZstdEncoder.cpp:250-340), whose units would run one behind the other.  The test is
// deliberately easy to pass: a frame taken by stage J for nothing costs several times the units' time, a chain left to the units
// orders of magnitude more
// (binaries compressed at level >= 3 split their blocks and copy by repcodes: only two units in three show the dependency in their first block).
__global__ void zstd_dec_frame_sizes_kernel(DecFrame* frames, uint32_t nFrames, DecBlock* __restrict__ blocks, DecCounts* counts, uint32_t jumpMode) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFrames) return;
    uint64_t total = 0; uint32_t st = 0, chained = 0, run = 0, longest = 0;
    const uint32_t b0 = frames[f].firstBlock, nb = frames[f].nBlocks;
    uint32_t r0 = 1, r1 = 4, r2 = 8;                                         // the format's starting history
    for (uint32_t i = 0; i < nb; i++) {
        DecBlock& B = blocks[b0 + i];
        B.outRel = total; B.repInit[0] = r0; B.repInit[1] = r1; B.repInit[2] = r2;
        total += B.regen; st |= B.status;
        if (B.regen > block_max(frames[f].windowSize)) st |= B2Z_DERR_CORRUPT;                // a compressed block decodes to at most Block_Maximum_Size
        if (i && i % B2Z_DEC_UNIT_BLOCKS == 0u) {                             // a unit's first block: does it copy from the unit before it?
            if (B.type == 2 && B.nearBehind) { chained++; run++; if (run > longest) longest = run; } else run = 0;
        }
        if (B.type == 2 && B.nbSeq) {                                         // apply the block's symbolic history (stage D1)
            const uint32_t in[3] = { r0, r1, r2 }, y = B.repSym;
            r0 = (y & 3u) ? in[(y & 3u) - 1u] - B.repX[0] : B.repX[0];
            r1 = ((y >> 2) & 3u) ? in[((y >> 2) & 3u) - 1u] - B.repX[1] : B.repX[1];
            r2 = ((y >> 4) & 3u) ? in[((y >> 4) & 3u) - 1u] - B.repX[2] : B.repX[2];
        }
    }
    if (frames[f].contentSize != ~0ull && frames[f].contentSize != total) st |= B2Z_DERR_CORRUPT;
    frames[f].regen = total;
    const uint32_t units = (nb + B2Z_DEC_UNIT_BLOCKS - 1u) / B2Z_DEC_UNIT_BLOCKS;
    frames[f].jump = (uint32_t)(!st && total &&
                                (jumpMode == 2u || (jumpMode == 1u && units >= B2Z_DEC_JUMP_MIN_UNITS && (longest >= 3u || chained * 4u >= (units - 1u) * 3u))));
    if (st) atomicOr(&counts->status, st);
}
__global__ void zstd_dec_frame_offsets_kernel(DecFrame* frames, uint32_t nFrames, uint64_t dstCap, DecCounts* counts, uint64_t* total) {
    if (threadIdx.x || blockIdx.x) return;
    uint64_t o = 0; uint32_t u = 0, nj = 0;
    for (uint32_t f = 0; f < nFrames; f++) {
        frames[f].dstOff = o; o += frames[f].regen;
        nj += frames[f].jump;
        frames[f].pad = u; if (!frames[f].jump) u += (frames[f].nBlocks + B2Z_DEC_UNIT_BLOCKS - 1u) / B2Z_DEC_UNIT_BLOCKS;
    }
    *total = o; counts->nUnits = u; counts->nJump = nj;
    if (o > dstCap) atomicOr(&counts->status, B2Z_DERR_DSTSIZE);
}

// ---------------------------------------------------------------- D3: execute
// One warp per UNIT of B2Z_DEC_UNIT_BLOCKS consecutive blocks of a frame (a frame of up to 1 MiB is one unit).  Units are taken from
// a ticket counter, so a running unit only ever has lower-numbered units running or finished beside it; stage D2 gave every block its
// output offset and its starting repcode history, so a unit needs nothing from its predecessors but the BYTES its matches copy.
// A match whose source starts before the unit's first byte waits for the done flag of the unit(s) that write those bytes -- in the
// frames of this encoder's long mode that is a far match into a region finished long ago; in a frame with a sliding window the
// units simply run one behind the other, as one warp per frame did.
// Inside a unit, blocks in order; sequences are taken 32 at a time (one per lane):
//   1. repcode history is resolved in order (warp-uniform registers) -> every lane knows its offset;
//   2. prefix sums give every lane its output position and literal source;
//   3. all literal runs are copied in parallel;
//   4. every match whose source ends before the batch's first output byte is copied in parallel;
//   5. the remaining matches (source overlaps this batch's output) are copied in sequence order,
//      each as a periodic extension (dst[i] = src[i mod offset]) so its bytes are independent.
__device__ __forceinline__ void warp_copy_match(uint8_t* dst, uint32_t offset, uint32_t n, uint32_t lane) {
    const uint8_t* m = dst - offset;
    if (offset >= n) { for (uint32_t i = lane; i < n; i += 32) dst[i] = __ldcg(m + i); }
    else { for (uint32_t i = lane; i < n; i += 32) dst[i] = __ldcg(m + (i % offset)); }
}
// index (within the frame) of the block that writes frame byte `pos`
__device__ __forceinline__ uint32_t dec_block_of(const DecBlock* __restrict__ fb, uint32_t nb, uint64_t pos) {
    uint32_t k = (uint32_t)(pos >> 17);                                       // exact while every earlier block is full
    if (k < nb && fb[k].outRel <= pos && pos < fb[k].outRel + fb[k].regen) return k;
    uint32_t lo = 0, hi = nb;                                                 // last block with outRel <= pos
    while (hi - lo > 1u) { const uint32_t mid = (lo + hi) >> 1; if (fb[mid].outRel <= pos) lo = mid; else hi = mid; }
    return lo;
}

__global__ void __launch_bounds__(32)
zstd_dec_exec_kernel(const uint8_t* __restrict__ src, DecFrame* __restrict__ frames, uint32_t nFrames, DecBlock* __restrict__ blocks,
                     const uint8_t* __restrict__ lits, const uint64_t* __restrict__ seqs, uint8_t* dst, DecCounts* counts, uint32_t* unitState) {
    if (counts->status) return;                                  // a failed stage: nothing is written (and nobody waits)
    // the last B2Z_DEC_RING output bytes of this warp, position p at ring[p % B2Z_DEC_RING]: a match that copies bytes of its own batch
    // (step 5) finds them here after a shared-memory round trip instead of a store-to-L2 / load-from-L2 one.  Batches that write more
    // than half the ring bypass it; ringFrom = first frame position from which the ring mirrors the output without gaps.
    __shared__ uint8_t ring[B2Z_DEC_RING];
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t nUnits = counts->nUnits;
    volatile uint32_t* done = unitState + 1;
    for (;;) {
        uint32_t u = 0;
        if (lane == 0) u = atomicAdd(unitState, 1u);
        u = __shfl_sync(B2Z_FULL, u, 0);
        if (u >= nUnits) break;
        uint32_t f;                                              // the frame of unit u: last frame with first unit <= u that has blocks
        { uint32_t lo = 0, hi = nFrames; while (hi - lo > 1u) { const uint32_t mid = (lo + hi) >> 1; if (frames[mid].pad <= u) lo = mid; else hi = mid; } f = lo; }
        const DecFrame fr = frames[f];
        const DecBlock* __restrict__ fblk = blocks + fr.firstBlock;
        const uint32_t k0 = (u - fr.pad) * B2Z_DEC_UNIT_BLOCKS, k1 = k0 + B2Z_DEC_UNIT_BLOCKS < fr.nBlocks ? k0 + B2Z_DEC_UNIT_BLOCKS : fr.nBlocks;
        uint8_t* out = dst + fr.dstOff;
        const uint64_t unitStart = fblk[k0].outRel;
        uint64_t o = unitStart;                                  // frame bytes produced before the next sequence
        uint64_t ringFrom = unitStart;
        uint32_t rep0 = fblk[k0].repInit[0], rep1 = fblk[k0].repInit[1], rep2 = fblk[k0].repInit[2], err = 0;
        for (uint32_t bi = fr.firstBlock + k0; bi < fr.firstBlock + k1 && !err; bi++) {
            const DecBlock blk = blocks[bi];
            if (blk.type == 0) { for (uint32_t i = lane; i < blk.rawSize; i += 32) out[o + i] = src[blk.srcOff + i]; o += blk.rawSize; ringFrom = o; __syncwarp(); continue; }
            if (blk.type == 1) { const uint8_t v = src[blk.srcOff]; for (uint32_t i = lane; i < blk.rawSize; i += 32) out[o + i] = v; o += blk.rawSize; ringFrom = o; __syncwarp(); continue; }
            const uint8_t* lit = lits + (size_t)blk.slot * 131072u;
            const uint64_t* sq = seqs + (size_t)blk.slot * B2Z_DEC_MAXSEQ;
            uint32_t lp = 0;
            uint64_t ahead = lane < blk.nbSeq ? sq[lane] : 0ull;                             // the next batch's sequences are fetched a batch ahead
            for (uint32_t i0 = 0; i0 < blk.nbSeq && !err; i0 += 32) {
                const uint32_t cnt = (blk.nbSeq - i0) < 32u ? (blk.nbSeq - i0) : 32u;
                const uint64_t mine = ahead;
                ahead = i0 + 32u + lane < blk.nbSeq ? sq[i0 + 32u + lane] : 0ull;
                const uint32_t ll = lane < cnt ? ((uint32_t)(mine >> 30) & 0x1FFFFu) : 0u;
                const uint32_t ml = lane < cnt ? ((uint32_t)(mine >> 47) + 3u) : 0u;
                // 1. repcodes.  A batch without repcode sequences (offBase > 3 everywhere: the usual case) needs no walk: every offset is
                //    explicit and the history is the last three of them; otherwise in order (ZSTD_decodeSequence's rules,
                //    zstd_decompress_block.c:1290-1312)
                uint32_t myOff = 0;
                const uint32_t obMine = (uint32_t)mine & 0x3FFFFFFFu;
                if (!__any_sync(B2Z_FULL, lane < cnt && obMine <= 3u)) {
                    myOff = lane < cnt ? obMine - 3u : 0u;
                    const uint32_t o1 = __shfl_sync(B2Z_FULL, myOff, cnt - 1u), o2 = __shfl_sync(B2Z_FULL, myOff, (cnt - 2u) & 31u), o3 = __shfl_sync(B2Z_FULL, myOff, (cnt - 3u) & 31u);
                    const uint32_t n2 = cnt >= 2u ? o2 : rep0, n3 = cnt >= 3u ? o3 : (cnt == 2u ? rep0 : rep1);
                    rep2 = n3; rep1 = n2; rep0 = o1;
                } else for (uint32_t k = 0; k < cnt; k++) {
                    const uint64_t s = __shfl_sync(B2Z_FULL, mine, k);
                    const uint32_t ob = (uint32_t)s & 0x3FFFFFFFu, llk = (uint32_t)(s >> 30) & 0x1FFFFu;
                    uint32_t offset;
                    if (ob > 3) { offset = ob - 3u; rep2 = rep1; rep1 = rep0; rep0 = offset; }
                    else {
                        const uint32_t idx = ob - 1u + (llk == 0u);
                        if (idx == 0) offset = rep0;
                        else {
                            offset = idx == 3 ? rep0 - 1u : (idx == 1 ? rep1 : rep2);
                            if (idx != 1) rep2 = rep1;
                            rep1 = rep0; rep0 = offset;
                        }
                    }
                    if (lane == k) myOff = offset;
                }
                // 2. positions (relative to o, the frame bytes produced before this batch)
                uint32_t total, litTotal;
                const uint32_t excl = warp_excl_scan(ll + ml, lane, &total);
                const uint32_t litExcl = warp_excl_scan(ll, lane, &litTotal);
                const uint32_t relDst = excl + ll;
                const uint64_t myDst = o + relDst;                                       // frame-relative
                const bool bad = lane < cnt && (myOff == 0 || myOff > myDst || myOff > fr.windowSize);
                if (__any_sync(B2Z_FULL, bad)) { err = B2Z_DERR_CORRUPT; break; }
                // 2b. a source that starts before this unit's first byte: wait for the unit(s) that write it
                const bool behind = lane < cnt && myDst - myOff < unitStart;
                if (__any_sync(B2Z_FULL, behind)) {
                    if (behind) {
                        const uint64_t a = myDst - myOff, e = (a + ml < unitStart ? a + ml : unitStart) - 1u;
                        const uint32_t ua = fr.pad + dec_block_of(fblk, fr.nBlocks, a) / B2Z_DEC_UNIT_BLOCKS, ue = fr.pad + dec_block_of(fblk, fr.nBlocks, e) / B2Z_DEC_UNIT_BLOCKS;
                        for (uint32_t x = ua; x <= ue && x < u; x++) while (done[x] == 0u) __nanosleep(256);
                        __threadfence();
                    }
                    __syncwarp();
                }
                const bool useRing = total <= B2Z_DEC_RING / 2u;                           // (warp-uniform)
                // 3. literals.  The batch's literal bytes are contiguous in the literal buffer: lane = byte, 32 per round; byte t belongs to the
                //    sequence k with litExcl_k <= t < litExcl_k + ll_k (binary search over the lanes' prefix sums).  B2Z_DEC_ROUNDS rounds are
                //    taken together: all their loads are issued before the first store needs its byte, so the rounds cost one global
                //    round trip, not one each (they were 2/3 of this kernel's time: ~10 dependent round trips per 32 sequences)
                for (uint32_t t0 = 0; t0 < litTotal; t0 += 32u * B2Z_DEC_ROUNDS) {
                    uint8_t v[B2Z_DEC_ROUNDS];
#pragma unroll
                    for (uint32_t r = 0; r < B2Z_DEC_ROUNDS; r++) { const uint32_t t = t0 + r * 32u + lane; v[r] = t < litTotal ? lit[lp + t] : (uint8_t)0; }
#pragma unroll
                    for (uint32_t r = 0; r < B2Z_DEC_ROUNDS; r++) {
                        const uint32_t t = t0 + r * 32u + lane;
                        if (t0 + r * 32u >= litTotal) break;                                     // (warp-uniform)
                        uint32_t k = 0;
#pragma unroll
                        for (uint32_t st = 16; st; st >>= 1) { const uint32_t w = __shfl_sync(B2Z_FULL, litExcl, (k + st) & 31u); if (k + st < 32u && w <= t) k += st; }
                        const uint32_t base = __shfl_sync(B2Z_FULL, excl, k), le = __shfl_sync(B2Z_FULL, litExcl, k);
                        if (t < litTotal) { const uint64_t pos = o + base + (t - le); out[pos] = v[r]; if (useRing) ring[pos & (B2Z_DEC_RING - 1u)] = v[r]; }
                    }
                }
                // 4. matches that read only bytes produced before this batch: the same flattening over their bytes, the same grouping of rounds
                const bool indep = lane < cnt && (myDst - myOff + ml <= o);
                {
                    uint32_t indepTotal;
                    const uint32_t mExcl = warp_excl_scan(indep ? ml : 0u, lane, &indepTotal);
                    for (uint32_t u0 = 0; u0 < indepTotal; u0 += 32u * B2Z_DEC_ROUNDS) {
                        uint64_t pos[B2Z_DEC_ROUNDS]; uint32_t of[B2Z_DEC_ROUNDS]; uint8_t v[B2Z_DEC_ROUNDS];
#pragma unroll
                        for (uint32_t r = 0; r < B2Z_DEC_ROUNDS; r++) {
                            const uint32_t uu = u0 + r * 32u + lane;
                            uint32_t k = 0;
#pragma unroll
                            for (uint32_t st = 16; st; st >>= 1) { const uint32_t w = __shfl_sync(B2Z_FULL, mExcl, (k + st) & 31u); if (k + st < 32u && w <= uu) k += st; }
                            const uint32_t d = __shfl_sync(B2Z_FULL, relDst, k), me = __shfl_sync(B2Z_FULL, mExcl, k);
                            of[r] = __shfl_sync(B2Z_FULL, myOff, k); pos[r] = o + d + (uu - me);
                        }
#pragma unroll
                        for (uint32_t r = 0; r < B2Z_DEC_ROUNDS; r++) v[r] = u0 + r * 32u + lane < indepTotal ? __ldcg(out + pos[r] - of[r]) : (uint8_t)0;
#pragma unroll
                        for (uint32_t r = 0; r < B2Z_DEC_ROUNDS; r++)
                            if (u0 + r * 32u + lane < indepTotal) { out[pos[r]] = v[r]; if (useRing) ring[pos[r] & (B2Z_DEC_RING - 1u)] = v[r]; }
                    }
                }
                __syncwarp();
                // 5. the rest, in order
                for (uint32_t dep = __ballot_sync(B2Z_FULL, lane < cnt && !indep); dep; dep &= dep - 1u) {
                    const uint32_t k = (uint32_t)__ffs((int)dep) - 1u;
                    const uint64_t dk = __shfl_sync(B2Z_FULL, myDst, k);
                    const uint32_t ok = __shfl_sync(B2Z_FULL, myOff, k), mk = __shfl_sync(B2Z_FULL, ml, k);
                    if (useRing && ok <= B2Z_DEC_RING / 2u && dk - ok >= ringFrom) {       // the whole source is in the ring
                        const uint32_t sk = (uint32_t)(dk - ok);
                        for (uint32_t i = lane; i < mk; i += 32) {
                            const uint8_t v = ring[(sk + (ok >= mk ? i : i % ok)) & (B2Z_DEC_RING - 1u)];
                            out[dk + i] = v; ring[((uint32_t)dk + i) & (B2Z_DEC_RING - 1u)] = v;
                        }
                    } else {
                        warp_copy_match(out + dk, ok, mk, lane);
                        if (useRing) { __syncwarp(); for (uint32_t i = lane; i < mk; i += 32) ring[((uint32_t)dk + i) & (B2Z_DEC_RING - 1u)] = __ldcg(out + dk + i); }
                    }
                    __syncwarp();
                }
                if (!useRing) ringFrom = o + total;
                o += total; lp += litTotal;
            }
            if (!err) { const uint32_t tail = blk.litSize - lp; for (uint32_t i = lane; i < tail; i += 32) out[o + i] = lit[lp + i]; o += tail; if (tail) ringFrom = o; }
            __syncwarp();
            if (!err && o != blk.outRel + blk.regen) err = B2Z_DERR_CORRUPT;              // the block wrote what stage D1 said it would
        }
        if (err && lane == 0) atomicOr(&counts->status, err);
        // every unit signals, failed or not: nobody waits for ever
        __threadfence();
        __syncwarp();
        if (lane == 0) atomicExch(unitState + 1 + u, 1u);
    }
}

// ---------------------------------------------------------------- stage J: frames resolved by pointer jumping
// A frame the reference's encoder wrote is ONE frame with a sliding window (zstdmt's jobs become blocks of one frame,
// zstdmt_compress.c:1403): every unit copies from the unit before it and stage D3 degrades to one chain.  Stage D1 has already
// decoded every sequence of every block and stage D2 placed every block, so the only thing left that is sequential is "a match
// copies bytes that a match before it produced" -- and that is a forest over the output bytes: a literal byte is a root, a match byte
// points at its source byte.  J1 writes the literal bytes and one pointer per output byte (one warp per block, all blocks at once);
// J2 doubles the pointers (ptr[i] = ptr[ptr[i]], in place: any value a neighbour holds meanwhile is an ancestor, so stale reads only
// cost a round) until every pointer names a literal -- ceil(log2(longest chain)) rounds of streaming passes; J3 fetches the bytes.
// The batch's output is taken in segments of at most 1 GiB, in order, so that a pointer fits 31 bits whatever the frame's size: a pointer is
// (position - segment start + 2^30) -- a source lies at most a window (<= 2^30 - 16) before its byte -- and bit 31 says "the byte there is
// final": a literal of this segment, or anything before the segment.
// Role in the reference: ZSTD_execSequence over the whole frame (zstd_decompress_block.c:1001-1100), which is strictly sequential.
__global__ void __launch_bounds__(128)
zstd_dec_jump_build_kernel(const uint8_t* __restrict__ src, const DecFrame* __restrict__ frames, const DecBlock* __restrict__ blocks, uint32_t nBlocks,
                           const uint8_t* __restrict__ lits, const uint64_t* __restrict__ seqs, uint8_t* __restrict__ dst, DecCounts* counts,
                           uint32_t* __restrict__ ptr, uint64_t segS, uint64_t segE) {
    if (counts->status) return;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t nWarps = (gridDim.x * blockDim.x) >> 5;
    // pointer of the byte at batch offset P (inside the segment): its own place if it is a literal, else its source Q; a source before the
    // segment is final already (earlier segments are complete)
    auto put = [&](uint64_t P, uint64_t Q, bool literal) {
        if (P < segS || P >= segE) return;
        ptr[P - segS] = (uint32_t)(Q + B2Z_DEC_JUMP_BIAS - segS) | ((literal || Q < segS) ? B2Z_DEC_JUMP_FINAL : 0u);
    };
    for (uint32_t bi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; bi < nBlocks; bi += nWarps) {
        const DecBlock blk = blocks[bi];
        const DecFrame* fp = frames + blk.frame;
        if (!fp->jump) continue;
        const uint64_t windowSize = fp->windowSize, fbase = fp->dstOff;          // batch offset of the frame's first byte
        if (fbase + blk.outRel >= segE || fbase + blk.outRel + blk.regen <= segS) continue;     // the block writes nothing into this segment
        uint64_t o = blk.outRel;                                             // frame bytes produced before the next sequence
        uint32_t err = 0;
        if (blk.type == 0) { for (uint32_t i = lane; i < blk.rawSize; i += 32) { const uint64_t P = fbase + o + i; if (P >= segS && P < segE) dst[P] = src[blk.srcOff + i]; put(P, P, true); } continue; }
        if (blk.type == 1) { const uint8_t v = src[blk.srcOff]; for (uint32_t i = lane; i < blk.rawSize; i += 32) { const uint64_t P = fbase + o + i; if (P >= segS && P < segE) dst[P] = v; put(P, P, true); } continue; }
        const uint8_t* __restrict__ lit = lits + (size_t)blk.slot * 131072u;
        const uint64_t* __restrict__ sq = seqs + (size_t)blk.slot * B2Z_DEC_MAXSEQ;
        uint32_t lp = 0, rep0 = blk.repInit[0], rep1 = blk.repInit[1], rep2 = blk.repInit[2];
        uint64_t ahead = lane < blk.nbSeq ? sq[lane] : 0ull;
        for (uint32_t i0 = 0; i0 < blk.nbSeq && !err; i0 += 32) {
            const uint32_t cnt = (blk.nbSeq - i0) < 32u ? (blk.nbSeq - i0) : 32u;
            const uint64_t mine = ahead;
            ahead = i0 + 32u + lane < blk.nbSeq ? sq[i0 + 32u + lane] : 0ull;
            const uint32_t ll = lane < cnt ? ((uint32_t)(mine >> 30) & 0x1FFFFu) : 0u;
            const uint32_t ml = lane < cnt ? ((uint32_t)(mine >> 47) + 3u) : 0u;
            // offsets: the repcode rules of stage D3 (zstd_decompress_block.c:1290-1312), history from stage D2
            uint32_t myOff = 0;
            const uint32_t obMine = (uint32_t)mine & 0x3FFFFFFFu;
            if (!__any_sync(B2Z_FULL, lane < cnt && obMine <= 3u)) {
                myOff = lane < cnt ? obMine - 3u : 0u;
                const uint32_t o1 = __shfl_sync(B2Z_FULL, myOff, cnt - 1u), o2 = __shfl_sync(B2Z_FULL, myOff, (cnt - 2u) & 31u), o3 = __shfl_sync(B2Z_FULL, myOff, (cnt - 3u) & 31u);
                const uint32_t n2 = cnt >= 2u ? o2 : rep0, n3 = cnt >= 3u ? o3 : (cnt == 2u ? rep0 : rep1);
                rep2 = n3; rep1 = n2; rep0 = o1;
            } else for (uint32_t k = 0; k < cnt; k++) {
                const uint64_t s = __shfl_sync(B2Z_FULL, mine, k);
                const uint32_t ob = (uint32_t)s & 0x3FFFFFFFu, llk = (uint32_t)(s >> 30) & 0x1FFFFu;
                uint32_t offset;
                if (ob > 3) { offset = ob - 3u; rep2 = rep1; rep1 = rep0; rep0 = offset; }
                else {
                    const uint32_t idx = ob - 1u + (llk == 0u);
                    if (idx == 0) offset = rep0;
                    else {
                        offset = idx == 3 ? rep0 - 1u : (idx == 1 ? rep1 : rep2);
                        if (idx != 1) rep2 = rep1;
                        rep1 = rep0; rep0 = offset;
                    }
                }
                if (lane == k) myOff = offset;
            }
            uint32_t total, litTotal;
            const uint32_t excl = warp_excl_scan(ll + ml, lane, &total);
            const uint32_t litExcl = warp_excl_scan(ll, lane, &litTotal);
            const uint64_t myDst = o + excl + ll;                                        // frame-relative start of the lane's match
            const bool bad = lane < cnt && (myOff == 0 || myOff > myDst || myOff > windowSize);
            if (__any_sync(B2Z_FULL, bad)) { err = B2Z_DERR_CORRUPT; break; }
            // lane = byte of the batch, B2Z_DEC_ROUNDS rounds of 32 taken together (their literal loads are issued before the first store);
            // byte t belongs to the sequence k with excl_k <= t < excl_k + ll_k + ml_k (binary search over the lanes' prefix sums)
            if (fbase + o < segE && fbase + o + total > segS)                            // (warp-uniform) the pass touches the segment
            for (uint32_t t0 = 0; t0 < total; t0 += 32u * B2Z_DEC_ROUNDS) {
                uint8_t v[B2Z_DEC_ROUNDS]; uint64_t w[B2Z_DEC_ROUNDS]; bool isLit[B2Z_DEC_ROUNDS];
#pragma unroll
                for (uint32_t r = 0; r < B2Z_DEC_ROUNDS; r++) {
                    const uint32_t t = t0 + r * 32u + lane;
                    uint32_t k = 0;
#pragma unroll
                    for (uint32_t st = 16; st; st >>= 1) { const uint32_t x = __shfl_sync(B2Z_FULL, excl, (k + st) & 31u); if (k + st < 32u && x <= t) k += st; }
                    const uint32_t e = __shfl_sync(B2Z_FULL, excl, k), l = __shfl_sync(B2Z_FULL, ll, k), le = __shfl_sync(B2Z_FULL, litExcl, k), of = __shfl_sync(B2Z_FULL, myOff, k);
                    const uint32_t rr = t - e;
                    v[r] = 0; w[r] = 0; isLit[r] = false;
                    if (t < total) {
                        if (rr < l) { v[r] = lit[lp + le + rr]; w[r] = fbase + o + t; isLit[r] = true; }
                        else {
                            // a match byte points at its source; inside an overlapping match (offset < length) at the byte of the period
                            // before the match, not at the match's own earlier byte: no chain inside one match
                            const uint32_t m = rr - l;
                            w[r] = fbase + o + e + l - of + (m < of ? m : m % of);
                        }
                    }
                }
#pragma unroll
                for (uint32_t r = 0; r < B2Z_DEC_ROUNDS; r++) {
                    const uint32_t t = t0 + r * 32u + lane;
                    if (t < total) { const uint64_t P = fbase + o + t; put(P, w[r], isLit[r]); if (isLit[r] && P >= segS && P < segE) dst[P] = v[r]; }
                }
            }
            o += total; lp += litTotal;
        }
        if (!err) {
            const uint32_t tail = blk.litSize - lp;
            for (uint32_t i = lane; i < tail; i += 32) { const uint64_t P = fbase + o + i; if (P >= segS && P < segE) dst[P] = lit[lp + i]; put(P, P, true); }
            o += tail;
            if (o != blk.outRel + blk.regen) err = B2Z_DERR_CORRUPT;
        }
        if (err && lane == 0) atomicOr(&counts->status, err);
    }
}

// the frame that holds batch offset i: the last frame with dstOff <= i (frames without output share their successor's offset)
__device__ __forceinline__ uint32_t dec_frame_of(const DecFrame* __restrict__ frames, uint32_t nFrames, uint64_t i) {
    uint32_t lo = 0, hi = nFrames;
    while (hi - lo > 1u) { const uint32_t mid = (lo + hi) >> 1; if (frames[mid].dstOff <= i) lo = mid; else hi = mid; }
    return lo;
}

// J2 (LAST = false): one round of pointer doubling over every jump frame's pointers; a warp takes 128 consecutive positions, four per lane.
// flags[r] = round r left a pointer that does not yet name a final byte; a round whose predecessor left none returns at once (all rounds are
// launched up front).  tileDone[w] = the 128 pointers of warp tile w are all final: later rounds read one byte instead of 512 (most of a round
// is streaming the pointer array, and after a few rounds most tiles have nothing left to do).
// J3 (LAST = true): dst[i] = dst[ptr[i]] for the match bytes.
template <bool LAST> __global__ void __launch_bounds__(256)
zstd_dec_jump_round_kernel(const DecFrame* __restrict__ frames, uint32_t nFrames, uint64_t segS, uint64_t segE, uint32_t* __restrict__ ptr, uint32_t* flags,
                           uint8_t* __restrict__ tileDone, uint32_t round, uint8_t* dst, DecCounts* counts) {
    if (counts->status) return;
    if (!LAST && round && !flags[round - 1u]) return;
    const uint64_t n = segE - segS, nTiles = (n + 127u) >> 7;
    const uint32_t lane = threadIdx.x & 31u;
    bool pending = false, broken = false;
    for (uint64_t tile = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; tile < nTiles; tile += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
        if (!LAST && tileDone[tile]) continue;                                       // (warp-uniform)
        const uint64_t i0 = (tile << 7) + (lane << 2);
        bool mine = false;                                                            // one of this lane's pointers is not final after this round
        if (i0 < n) {
            uint32_t f = nFrames > 1u ? dec_frame_of(frames, nFrames, segS + i0) : 0u;
            uint64_t fEnd = frames[f].dstOff + frames[f].regen; bool fj = frames[f].jump != 0u;
            uint4 q4 = *reinterpret_cast<const uint4*>(ptr + i0);
            uint32_t q[4] = { q4.x, q4.y, q4.z, q4.w }; bool take[4]; uint32_t r[4];
#pragma unroll
            for (uint32_t e = 0; e < 4; e++) {
                const uint64_t i = i0 + e;
                take[e] = false;
                if (i < n) {
                    while (segS + i >= fEnd) { f++; fEnd = frames[f].dstOff + frames[f].regen; fj = frames[f].jump != 0u; }
                    take[e] = fj && (LAST ? q[e] != (((uint32_t)i + B2Z_DEC_JUMP_BIAS) | B2Z_DEC_JUMP_FINAL) : !(q[e] & B2Z_DEC_JUMP_FINAL));
                }
            }
            if (!LAST) {
#pragma unroll
                for (uint32_t e = 0; e < 4; e++) r[e] = take[e] ? __ldcg(ptr + (q[e] - B2Z_DEC_JUMP_BIAS)) : q[e];   // not final: the source lies in this segment
                if (take[0] | take[1] | take[2] | take[3]) {
#pragma unroll
                    for (uint32_t e = 0; e < 4; e++) mine |= take[e] && !(r[e] & B2Z_DEC_JUMP_FINAL);
                    *reinterpret_cast<uint4*>(ptr + i0) = make_uint4(r[0], r[1], r[2], r[3]);
                }
            } else {
#pragma unroll
                for (uint32_t e = 0; e < 4; e++) {                                           // the source's batch offset: segS + pointer - bias (>= 0: a byte of the batch)
                    broken |= take[e] && !(q[e] & B2Z_DEC_JUMP_FINAL);
                    r[e] = take[e] ? dst[segS + (q[e] & ~B2Z_DEC_JUMP_FINAL) - B2Z_DEC_JUMP_BIAS] : 0u;
                }
#pragma unroll
                for (uint32_t e = 0; e < 4; e++) if (take[e]) dst[segS + i0 + e] = (uint8_t)r[e];
            }
        }
        if (!LAST) {
            pending |= mine;
            if (!__any_sync(B2Z_FULL, mine) && lane == 0) tileDone[tile] = 1;
        }
    }
    if (!LAST && pending) flags[round] = 1u;
    if (LAST && broken) atomicOr(&counts->status, B2Z_DERR_CORRUPT);       // a pointer no round resolved: cannot happen (pointers strictly decrease)
}

// ---------------------------------------------------------------- checksum verification
// one warp per frame (xxh64_warp: lanes 0-3 hash, the warp streams the frame through shared memory)
__global__ void __launch_bounds__(64)
zstd_dec_verify_kernel(const uint8_t* __restrict__ src, const DecFrame* __restrict__ frames, uint32_t nFrames,
                       const uint8_t* __restrict__ dst, DecCounts* counts) {
    __shared__ __align__(16) uint8_t tiles[2][B2Z_XXH_WS_BYTES];
    const uint32_t lane = threadIdx.x & 31u, wic = threadIdx.x >> 5;
    const uint32_t f = blockIdx.x * (blockDim.x >> 5) + wic;
    if (f >= nFrames || counts->status) return;
    const DecFrame fr = frames[f];
    if (!fr.checksum) return;
    const uint8_t* c = src + fr.endOff - 4;
    const uint32_t want = (uint32_t)c[0] | ((uint32_t)c[1] << 8) | ((uint32_t)c[2] << 16) | ((uint32_t)c[3] << 24);
    const uint64_t h = xxh64_warp(dst + fr.dstOff, fr.regen, tiles[wic], lane);        // frame outputs start at arbitrary byte offsets
    if (lane == 0 && (uint32_t)h != want) atomicOr(&counts->status, B2Z_DERR_CHECKSUM);
}

// ---------------------------------------------------------------- launchers
#ifndef B2Z_CUEMU
void launch_zstd_dec_verify(const uint8_t* src, const DecFrame* frames, uint32_t nFrames, const uint8_t* dst, DecCounts* counts, cudaStream_t st) {
    if (nFrames) zstd_dec_verify_kernel<<<(nFrames + 1) / 2, 64, 0, st>>>(src, frames, nFrames, dst, counts);
}
void launch_zstd_dec_find_frames(const uint8_t* src, uint64_t srcSize, DecFrame* frames, uint32_t frameCap, DecCounts* counts, bool useHints, cudaStream_t st) {
    zstd_dec_find_frames_kernel<<<1, 32, 0, st>>>(src, srcSize, frames, frameCap, counts, useHints ? 1u : 0u);
}
void launch_zstd_dec_index_blocks(const uint8_t* src, uint64_t srcSize, DecFrame* frames, uint32_t nFrames,
                                  DecBlock* blocks, uint32_t blockCap, DecCounts* counts, cudaStream_t st) {
    if (!nFrames) return;
    const uint32_t grid = (nFrames + 63) / 64;
    zstd_dec_count_blocks_kernel<<<grid, 64, 0, st>>>(src, srcSize, frames, nFrames, counts);
    zstd_dec_scan_blocks_kernel<<<1, 32, 0, st>>>(frames, nFrames, blockCap, counts);
    zstd_dec_fill_blocks_kernel<<<grid, 64, 0, st>>>(src, srcSize, frames, nFrames, blocks, blockCap, counts);
}
void launch_zstd_dec_entropy(const uint8_t* src, uint64_t srcSize, DecBlock* blocks, uint32_t nBlocks, uint8_t* lits, uint64_t* seqs,
                             void* scratch, uint32_t smCount, cudaStream_t st, cudaStream_t stLit, cudaEvent_t evFork, cudaEvent_t evJoin) {
    if (!nBlocks) return;
    // scratch layout: hufTabs [nBlocks][2048] u16 | seqTabs [nBlocks][1280] SeqEnt | litJobs | seqJobs
    uint8_t* p = (uint8_t*)scratch;
    uint16_t* hufTabs = (uint16_t*)p; p += (size_t)nBlocks * 4096u;
    SeqEnt* seqTabs = (SeqEnt*)p; p += (size_t)nBlocks * 1280u * sizeof(SeqEnt);
    LitJob* litJobs = (LitJob*)p; p += (size_t)nBlocks * sizeof(LitJob);
    SeqJob* seqJobs = (SeqJob*)p;
    // The literal and the sequence kernels only read src/blocks and write disjoint outputs, so they may run on two streams
    // (stLit != st).  The four kernels each fill the GPU, and co-scheduling them
    // only makes them evict each other's lines (two streams measured slower than one).
    // The host dispatcher therefore passes stLit == st.
    if (stLit != st) { cudaEventRecord(evFork, st); cudaStreamWaitEvent(stLit, evFork, 0); }
    const uint32_t cap = smCount * 16u;
    { uint32_t grid = (nBlocks + D1_WARPS(0) - 1) / D1_WARPS(0); if (grid > cap) grid = cap;
      zstd_dec_entropy_kernel<0><<<grid, D1_WARPS(0) * 32, 0, stLit>>>(src, srcSize, blocks, nBlocks, lits, hufTabs, litJobs, seqTabs, seqJobs);
      cudaFuncSetAttribute(zstd_dec_lit_streams_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(B2Z_LIT_BLOCKS * 4096u));
      zstd_dec_lit_streams_kernel<<<(nBlocks + B2Z_LIT_BLOCKS - 1u) / B2Z_LIT_BLOCKS, B2Z_LIT_BLOCKS * 4u, B2Z_LIT_BLOCKS * 4096u, stLit>>>(src, srcSize, blocks, nBlocks, lits, hufTabs, litJobs); }
    { uint32_t grid = (nBlocks + D1_WARPS(1) - 1) / D1_WARPS(1); if (grid > cap) grid = cap;
      zstd_dec_entropy_kernel<1><<<grid, D1_WARPS(1) * 32, 0, st>>>(src, srcSize, blocks, nBlocks, lits, hufTabs, litJobs, seqTabs, seqJobs);
      zstd_dec_seq_streams_kernel<<<(nBlocks + 127u) / 128u, 128, 0, st>>>(src, srcSize, blocks, nBlocks, seqs, seqTabs, seqJobs); }
    if (stLit != st) { cudaEventRecord(evJoin, stLit); cudaStreamWaitEvent(st, evJoin, 0); }
}
size_t zstd_dec_entropy_scratch_bytes(uint32_t nBlocks) { return (size_t)nBlocks * (4096u + 1280u * sizeof(SeqEnt) + sizeof(LitJob) + sizeof(SeqJob)) + 256u; }
void launch_zstd_dec_layout(DecFrame* frames, uint32_t nFrames, DecBlock* blocks, uint64_t dstCap, DecCounts* counts, uint64_t* total, uint32_t jumpMode, cudaStream_t st) {
    if (nFrames) zstd_dec_frame_sizes_kernel<<<(nFrames + 127) / 128, 128, 0, st>>>(frames, nFrames, blocks, counts, jumpMode);
    zstd_dec_frame_offsets_kernel<<<1, 32, 0, st>>>(frames, nFrames, dstCap, counts, total);
}
size_t zstd_dec_jump_scratch_bytes(uint64_t total, uint32_t segLog) {         // flags | pointers of one segment | one byte per 128 pointers
    const uint64_t seg = total < (1ull << segLog) ? total : (1ull << segLog);
    return 256 + ((size_t)seg + 16) * 4 + (size_t)((seg + 127) >> 7) + 64;
}
void launch_zstd_dec_jump(const uint8_t* src, DecFrame* frames, uint32_t nFrames, DecBlock* blocks, uint32_t nBlocks, const uint8_t* lits, const uint64_t* seqs,
                          uint8_t* dst, uint64_t total, uint32_t segLog, DecCounts* counts, void* scratch, uint32_t smCount, cudaStream_t st) {
    if (!nFrames || !nBlocks || !total) return;
    const uint64_t seg = 1ull << segLog, segWords = total < seg ? total : seg;
    uint32_t* flags = (uint32_t*)scratch; uint32_t* ptr = (uint32_t*)((uint8_t*)scratch + 256);
    uint8_t* tileDone = (uint8_t*)(ptr + segWords + 16);
    const uint32_t cap = smCount * 16u;
    for (uint64_t S = 0; S < total; S += seg) {                        // segments in order: what lies before a segment is complete
        const uint64_t E = S + seg < total ? S + seg : total;
        cudaMemsetAsync(flags, 0, (B2Z_DEC_JUMP_ROUNDS + 1u) * 4u, st);
        cudaMemsetAsync(tileDone, 0, (size_t)((E - S + 127) >> 7), st);
        { const uint32_t want = (nBlocks + 3u) / 4u, grid = want < cap ? want : cap;
          zstd_dec_jump_build_kernel<<<grid, 128, 0, st>>>(src, frames, blocks, nBlocks, lits, seqs, dst, counts, ptr, S, E); }
        const uint64_t groups = (E - S + 3u) >> 2;
        const uint32_t grid = (uint32_t)((groups + 255u) / 256u < cap ? (groups + 255u) / 256u : cap);
        for (uint32_t r = 0; r < B2Z_DEC_JUMP_ROUNDS; r++) zstd_dec_jump_round_kernel<false><<<grid, 256, 0, st>>>(frames, nFrames, S, E, ptr, flags, tileDone, r, dst, counts);
        zstd_dec_jump_round_kernel<true><<<grid, 256, 0, st>>>(frames, nFrames, S, E, ptr, flags, tileDone, 0, dst, counts);
    }
}
size_t zstd_dec_unit_state_bytes(uint32_t nFrames, uint32_t nBlocks) { return ((size_t)nBlocks / B2Z_DEC_UNIT_BLOCKS + nFrames + 2u) * 4u; }
void launch_zstd_dec_exec(const uint8_t* src, DecFrame* frames, uint32_t nFrames, DecBlock* blocks, uint32_t nBlocks, const uint8_t* lits, const uint64_t* seqs,
                          uint8_t* dst, DecCounts* counts, uint32_t* unitState, uint32_t smCount, cudaStream_t st) {
    if (!nFrames) return;
    cudaMemsetAsync(unitState, 0, zstd_dec_unit_state_bytes(nFrames, nBlocks), st);
    const uint32_t maxUnits = nBlocks / B2Z_DEC_UNIT_BLOCKS + nFrames;          // every frame rounds up once
    const uint32_t resident = smCount * 32u, grid = maxUnits < resident ? maxUnits : resident;        // resident warps; the others' units are taken by whoever finishes
    zstd_dec_exec_kernel<<<grid, 32, 0, st>>>(src, frames, nFrames, blocks, lits, seqs, dst, counts, unitState);
}
#endif

}  // namespace b2z
