// zstd_dec.cu -- Zstandard decoder kernels (sm_90a), bit-exact for any valid frame whose
// window is <= 2^29 and that needs no dictionary.
//
//   D0 prepass  (1 thread)          walk frame and block headers (sequential by format), record
//                                   per block where its entropy tables come from (treeless
//                                   literals / repeat-mode FSE tables chain back to an earlier block)
//   D1 entropy  (thread / stream)   Huffman-decode the literals (4 streams -> 4 threads) and FSE-decode
//                                   the sequences (one backward bitstream -> 1 thread), tables in shared memory
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
// The frame and block header walk is b2z_dec.h's.  D0 has the whole stream, so a frame cut short is corrupt; what makes a frame
// unsupported was met before any fault of its header (the parse stops at the first), so it comes first.
__device__ __forceinline__ uint32_t d0_status(uint32_t walk) { return walk == B2Z_DERR_TRUNCATED ? B2Z_DERR_CORRUPT : walk; }
__device__ __forceinline__ uint32_t d0_frame_status(const ZstdFrameHdr& h) { return h.unsupported ? h.unsupported : d0_status(h.status); }

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
        uint64_t sz;
        if (zstd_skippable(S, magic, ip, srcSize, &sz)) {
            if (srcSize - ip < sz) { status = B2Z_DERR_CORRUPT; break; }
            // a size hint? (payload = compressed size of the zstd frame that follows; verified by D0b)
            if (useHints && magic == 0x184D2A50u && sz == 12 && srcSize - ip >= 16 && S.le32(ip + 12) == B2Z_ZSTD_MAGIC) {
                const uint64_t fsz = S.le32(ip + 8);
                if (fsz >= 9 && srcSize - (ip + 12) >= fsz) {
                    if (nf >= frameCap) { status = B2Z_DERR_TABLE_FULL; break; }
                    DecFrame fr; fr.srcOff = ip + 12; fr.dstOff = 0; fr.contentSize = ~0ull; fr.windowSize = 0; fr.regen = ip + 12 + fsz;   // regen: end offset (until D2)
                    fr.firstBlock = 0; fr.nBlocks = 0; fr.checksum = 0; fr.pad = 1; fr.endOff = ip + 12 + fsz; fr.jump = 0; fr.nComp = 0; fr.firstSlot = 0; fr.pad4 = 0;                          // pad: 1 = end offset is a hint
                    frames[nf++] = fr; hinted++;
                    ip += 12 + fsz; continue;
                }
            }
            ip += sz; continue;
        }
        if (magic != B2Z_ZSTD_MAGIC) { status = B2Z_DERR_CORRUPT; break; }
        if (nf >= frameCap) { status = B2Z_DERR_TABLE_FULL; break; }
        const ZstdFrameHdr h = zstd_frame_hdr(S, ip, srcSize);
        if ((status = d0_frame_status(h))) break;
        const ZstdBlocks w = zstd_walk_blocks(S, ip, srcSize, h, ZstdEmitNone{});
        if ((status = d0_status(w.status))) break;
        DecFrame fr; fr.srcOff = ip; fr.dstOff = 0; fr.contentSize = ~0ull; fr.windowSize = 0; fr.regen = w.end; fr.firstBlock = 0; fr.nBlocks = w.nBlocks; fr.checksum = 0; fr.pad = 0; fr.endOff = w.end; fr.jump = 0; fr.nComp = 0; fr.firstSlot = 0; fr.pad4 = 0;
        frames[nf++] = fr;
        ip = w.end;
    }
    counts->nFrames = nf; counts->nBlocks = 0; counts->status = status; counts->srcUsed = ip; counts->nUnits = hinted;
}

__global__ void zstd_dec_count_blocks_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecFrame* frames, uint32_t nFrames, DecCounts* counts) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFrames) return;
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    DecFrame fr = frames[f];
    const ZstdFrameHdr h = zstd_frame_hdr(S, fr.srcOff, srcSize);
    uint32_t status = d0_frame_status(h), nb = 0, nComp = 0;
    if (!status) {
        const ZstdBlocks w = zstd_walk_blocks(S, fr.srcOff, srcSize, h, [&](uint32_t, uint32_t type, uint32_t, uint64_t, uint32_t) { nComp += type == 2; return 0u; });
        if ((status = d0_status(w.status))) nComp = 0;
        else {
            nb = w.nBlocks;
            if (w.end != fr.regen) status = B2Z_DERR_CORRUPT;           // a size hint that does not match its frame
        }
    }
    fr.contentSize = h.contentSize; fr.windowSize = h.windowSize; fr.checksum = h.checksum; fr.nBlocks = nb; fr.nComp = nComp;
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

// The block table entries of one frame, and where each compressed block's entropy tables come from: treeless literals reuse the
// frame's last Huffman table, repeat mode its last FSE table of the kind.
__global__ void zstd_dec_fill_blocks_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecFrame* frames, uint32_t nFrames,
                                            DecBlock* blocks, uint32_t blockCap, DecCounts* counts) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFrames || counts->status) return;
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    const DecFrame fr = frames[f];
    uint32_t nComp = 0; int32_t lastHuf = -1, lastTbl[3] = { -1, -1, -1 };
    const ZstdFrameHdr h = zstd_frame_hdr(S, fr.srcOff, srcSize);
    const ZstdBlocks w = zstd_walk_blocks(S, fr.srcOff, srcSize, h, [&](uint32_t k, uint32_t type, uint32_t bsize, uint64_t ip, uint32_t cSize) -> uint32_t {
        if (fr.firstBlock + k >= blockCap) return B2Z_DERR_TABLE_FULL;
        const int32_t self = (int32_t)(fr.firstBlock + k);
        DecBlock b; b.srcOff = ip; b.type = type; b.frame = f; b.hufSrc = -1; b.tblSrc[0] = b.tblSrc[1] = b.tblSrc[2] = -1;
        b.regen = 0; b.nbSeq = 0; b.litSize = 0; b.status = 0; b.rawSize = 0; b.cSize = cSize; b.nearBehind = 0;
        b.slot = type == 2 ? fr.firstSlot + nComp++ : 0xFFFFFFFFu; b.pad4 = 0;              // only compressed blocks own literal / sequence scratch
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
        blocks[self] = b;
        return 0u;
    });
    frames[f].regen = 0; frames[f].pad = 0;
    if (w.status) atomicOr(&counts->status, d0_status(w.status));
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

// ---------------------------------------------------------------- D1 tables (built on chip, one thread per block)
// Sequence decoding tables of one block: LL [0,512) | OF [512,768) | ML [768,1280) entries of 16 bits, symbol | ns << 6, where ns
// is FSE_buildDTable's per-symbol state counter (< 2^10): the state's nbBits = log - highbit(ns) and its next-state base =
// (ns << nbBits) - 2^log.  The baseline and the number of extra bits follow from the symbol (k_seqSym below for LL and ML;
// 1 << s and s for OF).  Two bytes per state keep 2.5 KiB per block in shared memory.
#define B2Z_SEQ_TAB 1280u
__device__ __forceinline__ uint32_t seq_tab_off(int t) { return t == 0 ? 0u : (t == 1 ? 512u : 768u); }

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

// FSE decoding table into tab[0, 2^log) (seq_tab_off's layout); norm[] is consumed (it ends as the state counters).  false when
// the spread does not close (malformed counts)
__device__ bool build_seq_table(uint16_t* tab, int16_t* norm, uint32_t maxSym, uint32_t log) {
    const uint32_t size = 1u << log, mask = size - 1u; uint32_t high = size - 1u;
    for (uint32_t s = 0; s <= maxSym; s++) if (norm[s] == -1) tab[high--] = (uint16_t)s;
    const uint32_t step = (size >> 1) + (size >> 3) + 3u; uint32_t pos = 0;
    for (uint32_t s = 0; s <= maxSym; s++)
        for (int i = 0; i < norm[s]; i++) { tab[pos] = (uint16_t)s; pos = (pos + step) & mask; while (pos > high) pos = (pos + step) & mask; }
    if (pos != 0) return false;
    for (uint32_t s = 0; s <= maxSym; s++) if (norm[s] == -1) norm[s] = 1;
    for (uint32_t u = 0; u < size; u++) { const uint32_t s = tab[u], ns = (uint32_t)norm[s]++; tab[u] = (uint16_t)(s | (ns << 6)); }
    return true;
}

// Walk the table descriptions of block `blk`'s sequences section; returns the offset (absolute in src)
// and mode of type t's description.  false on malformed data.  norm: scratch of 53 counts
__device__ bool locate_seq_table(const Src& S, const DecBlock& blk, int t, int16_t* norm, uint64_t* descOff, uint32_t* mode, uint32_t* avail) {
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
        else if (m == 2) { uint32_t ms = maxSymT[k], lg; used = fse_read_ncount(norm, &ms, &lg, S, p, left, maxLogT[k]); if (!used) return false; }
        if (used > left) return false;
        p += used; left -= used;
    }
    return false;
}

// Huffman weights of the description at `off` into w[0, *nw) (the last, implied weight included), checked as a complete code;
// returns the description's bytes and *maxBits, or 0.  One thread; its scratch lives in its own frame.
__device__ __forceinline__ uint32_t huf_read_weights(uint8_t* w, uint32_t* nwOut, uint32_t* maxBitsOut, const Src& S, uint64_t off, uint32_t size) {
    if (size < 1) return 0;
    uint32_t nw = 0;
    const uint32_t hb = S.u8(off); uint32_t used;
    if (hb >= 128) {
        nw = hb - 127u; used = 1u + (nw + 1u) / 2u;
        if (used > size) return 0;
        for (uint32_t i = 0; i < nw; i++) { const uint32_t v = S.u8(off + 1 + i / 2); w[i] = (uint8_t)((i & 1u) ? (v & 15u) : (v >> 4)); }
    } else {
        used = 1u + hb;
        if (hb == 0 || used > size) return 0;
        int16_t norm[256]; uint16_t nxt[256];
        uint32_t maxSym = 255, al;
        const uint32_t hs = fse_read_ncount(norm, &maxSym, &al, S, off + 1, hb, 6);
        if (!hs || hs >= hb) return 0;
        // the weights' FSE table (at most 64 states): symbol per state, nbBits | newState << 8
        uint8_t fsym[64]; uint16_t fdt[64];
        {
            const uint32_t size2 = 1u << al, mask = size2 - 1u; uint32_t high = size2 - 1u;
            for (uint32_t s = 0; s <= maxSym; s++) { if (norm[s] == -1) { fsym[high--] = (uint8_t)s; nxt[s] = 1; } else nxt[s] = (uint16_t)norm[s]; }
            const uint32_t step = (size2 >> 1) + (size2 >> 3) + 3u; uint32_t pos = 0;
            for (uint32_t s = 0; s <= maxSym; s++)
                for (int i = 0; i < norm[s]; i++) { fsym[pos] = (uint8_t)s; pos = (pos + step) & mask; while (pos > high) pos = (pos + step) & mask; }
            if (pos != 0) return 0;
            for (uint32_t u = 0; u < size2; u++) {
                const uint32_t s = fsym[u], ns = nxt[s]++;
                const uint32_t nbb = al - highbit32(ns);
                fdt[u] = (uint16_t)(nbb | ((((ns << nbb) - size2) & 0xFFu) << 8));     // newState < 64
            }
        }
        BwdBits b; if (b.init(&S, off + 1 + hs, hb - hs)) return 0;
        uint32_t s1 = b.read(al), s2 = b.read(al);
        if (b.overflow) return 0;
        for (;;) {
            if (nw > 253) return 0;
            w[nw++] = fsym[s1]; { const uint32_t e = fdt[s1]; s1 = (e >> 8) + b.read(e & 255u); }
            if (b.overflow) { w[nw++] = fsym[s2]; break; }
            if (nw > 253) return 0;
            w[nw++] = fsym[s2]; { const uint32_t e = fdt[s2]; s2 = (e >> 8) + b.read(e & 255u); }
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
    *nwOut = nw; *maxBitsOut = maxBits;
    return used;
}

// Fill the 2^maxBits-entry decoding table (symbol | nbBits << 8) from checked weights: the symbols of weight r take
// consecutive runs of 2^(r-1) entries from the weight class's start.  Thread k of n writes the entries i = k (mod n) of
// every run.
__device__ void huf_fill(uint16_t* huf, const uint8_t* w, uint32_t nw, uint32_t maxBits, uint32_t k, uint32_t n) {
    uint32_t rank[13], start[13];
    for (uint32_t r = 0; r < 13; r++) rank[r] = 0;
    for (uint32_t i = 0; i < nw; i++) rank[w[i]]++;
    uint32_t pos = 0;
    for (uint32_t r = 1; r <= maxBits; r++) { start[r] = pos; pos += rank[r] << (r - 1u); }
    for (uint32_t s = 0; s < nw; s++) {
        const uint32_t r = w[s]; if (!r) continue;
        const uint32_t len = 1u << (r - 1u); const uint16_t e = (uint16_t)(s | ((maxBits + 1u - r) << 8));
        for (uint32_t i = k; i < len; i += n) huf[start[r] + i] = e;
        start[r] += len;
    }
}
// Hot-loop reader (32-bit arithmetic): `cont` holds stream bytes [bytePos, bytePos+8); the next unread bit is
// bit (63 - consumed) of it.  After reload() consumed <= 7, so 57 bits can be read before the next reload.
// Bytes below the stream start read as zero; left() < 0 means the stream was over-read.
//
// No reload waits for memory.  `cont` is built with a funnel shift from the two aligned source words that hold it (lo = word wi,
// hi = word wi + 1, in registers).  The B2Z_BWD_DEPTH words below them are in flight to the thread's ring in shared memory
// (`ring`, B2Z_BWD_DEPTH words, word k in slot k mod B2Z_BWD_DEPTH): when the window crosses into the next word down, that word is
// taken from the ring and the one B2Z_BWD_DEPTH further down is asked for (cp.async, zero-filled for indices outside the source,
// which are never read).  A load is so first used about B2Z_BWD_DEPTH * 8 stream bytes after it was issued.  A reader's words
// still in flight are waited for by its next init() and by drain().
#define B2Z_BWD_DEPTH 4u
struct FastBwd {
    const Src* S; uint64_t* ring; uint64_t cont, lo, hi; int64_t wi; int32_t bytePos; uint32_t consumed, o;     // o = (start of cont) & 7
    __device__ __forceinline__ uint64_t word(int64_t k) const { return k >= 0 ? S->word((uint64_t)k) : 0ull; }
    __device__ __forceinline__ void issue(int64_t k) {                                      // word k into its ring slot
        uint64_t* d = ring + ((uint32_t)k & (B2Z_BWD_DEPTH - 1u));
#ifndef B2Z_CUEMU
        const bool in = k >= 0 && (uint64_t)k < S->nWords;
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n\tcp.async.commit_group;" ::
                     "r"((uint32_t)__cvta_generic_to_shared(d)), "l"(S->w + (in ? k : 0)), "r"(in ? 8u : 0u) : "memory");
#else
        *d = word(k);
#endif
    }
    __device__ __forceinline__ void drain() const {
#ifndef B2Z_CUEMU
        asm volatile("cp.async.wait_all;" ::: "memory");
#endif
    }
    __device__ __forceinline__ void window() {                                              // cont from lo, hi; zero below the start
        cont = funnel64(lo, hi, o * 8u);
        if (bytePos < 0) cont = bytePos > -8 ? cont & (~0ull << ((uint32_t)(-bytePos) * 8u)) : 0ull;
    }
    __device__ __forceinline__ int init(const Src* s, uint64_t* r, uint64_t b, uint32_t size) {
        S = s; ring = r;
        if (!size) return -1;
        const uint32_t lastByte = S->u8(b + size - 1);
        if (!lastByte) return -1;
        bytePos = (int32_t)size - 8; consumed = 8u - highbit32(lastByte);      // skip the padding and the end mark
        const int64_t p = (int64_t)b + bytePos;
        wi = p >> 3; o = (uint32_t)p & 7u;
        drain();                                                                // the ring's slots are free
        lo = word(wi); hi = word(wi + 1);
        for (uint32_t d = 1; d <= B2Z_BWD_DEPTH; d++) issue(wi - d);
        window();
        return 0;
    }
    // The line 256 bytes below is also asked into L2 when a word is crossed, so that the ring's load that reaches it does not wait for
    // HBM.
    __device__ __forceinline__ void reload() {
        const uint32_t d = consumed >> 3;                                       // <= 8 bytes: at most one word is crossed
        bytePos -= (int32_t)d; consumed &= 7u;
        if (o < d) {
#ifndef B2Z_CUEMU
            asm volatile("cp.async.wait_group %0;" :: "n"(B2Z_BWD_DEPTH - 1u) : "memory");    // word wi - 1 has arrived
#endif
            wi--; hi = lo; lo = ring[(uint32_t)wi & (B2Z_BWD_DEPTH - 1u)];
            issue(wi - (int64_t)B2Z_BWD_DEPTH);
#ifndef B2Z_CUEMU
            if (bytePos >= 256 + 8) asm volatile("prefetch.L2 [%0];" :: "l"(S->w + (wi - 32)));
#endif
            o += 8u;
        }
        o -= d;
        window();
    }
    __device__ __forceinline__ uint32_t read(uint32_t n) {                      // n <= 32 (0 allowed)
        const uint32_t v = (uint32_t)(((cont << consumed) >> 1) >> (63u - n));
        consumed += n;
        return v;
    }
    __device__ __forceinline__ int32_t left() const { return bytePos * 8 + 64 - (int32_t)consumed; }   // unread bits
};

// ---------------------------------------------------------------- D1: entropy decode
// Four kernels, two per section, and no table ever leaves the SM:
//   zstd_dec_entropy_kernel<0>  (warp / block)    literal headers; raw / RLE literals are expanded here
//   zstd_dec_lit_streams_kernel (4 threads / block) builds the Huffman table in shared memory, one thread per stream decodes
//   zstd_dec_entropy_kernel<1>  (thread / block)  sequence headers: where the three table descriptions are (an earlier block's
//                                                 for repeat mode), their sizes checked; the bookkeeping of blocks without sequences
//   zstd_dec_seq_streams_kernel (thread / block)  builds the three FSE tables in shared memory and decodes the bitstream
// Each serial bitstream is decoded by ONE THREAD, so that thousands of dependent chains overlap.  A table is built from the
// description in src (an earlier block's for treeless literals and repeat mode: any block may be read, a CTA depends on no other
// CTA).  The stream kernels loop over their groups of blocks, so they do not depend on the grid they are given.
// -DB2Z_D1_CLOCKS (off by default; tools/dec_entropy_profile.py --build-clocks): every stream thread of the two stream kernels
// adds the clock64() cycles it spends in each phase -- table build, refills, table look-ups and arithmetic, output stores -- to
// d1_clocks[]; b200z_d1_clocks() reads and clears them.  Without the switch the ticks compile to nothing.
enum { D1C_TABLE, D1C_REFILL, D1C_DECODE, D1C_STORE, D1C_N };
#ifdef B2Z_D1_CLOCKS
__device__ unsigned long long d1_clocks[2 * D1C_N];                     // literal kernel's phases, then the sequence kernel's
#define D1_CLOCKS_START() unsigned long long d1c[D1C_N] = {}; long long d1Last = clock64()
#define D1_TICK(ph) do { const long long now_ = clock64(); d1c[ph] += (unsigned long long)(now_ - d1Last); d1Last = now_; } while (0)
#define D1_CLOCKS_FLUSH(kernel) do { for (int p_ = 0; p_ < D1C_N; p_++) atomicAdd(&d1_clocks[(kernel) * D1C_N + p_], d1c[p_]); } while (0)
#else
#define D1_CLOCKS_START() do { } while (0)
#define D1_TICK(ph) do { } while (0)
#define D1_CLOCKS_FLUSH(kernel) do { } while (0)
#endif

#define SEQ_PACK(ob, ll, ml) ((uint64_t)(ob) | ((uint64_t)(ll) << 30) | ((uint64_t)((ml) - 3u) << 47))

typedef uint16_t SeqEnt;                            // one state of a sequence decoding table (B2Z_SEQ_TAB layout above)
struct LitJob { uint64_t off; uint32_t size, regen, streams, type; };          // Huffman literals: the section after its header
struct SeqJob { uint64_t bsOff, desc[3]; uint32_t bsLeft, nbSeq, litRegen, modes, avail[3], pad; };  // table t: description, mode, bytes left
#define D1_WARPS(ROLE) ((ROLE) == 0 ? 6 : 4)
// The table arguments (hufTabs, seqTabs) are not used: the tables are built where they are read.
template <int ROLE> __global__ void __launch_bounds__(D1_WARPS(ROLE) * 32)
zstd_dec_entropy_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecBlock* __restrict__ blocks, uint32_t nBlocks,
                        uint8_t* __restrict__ lits, uint16_t* __restrict__ hufTabs, LitJob* __restrict__ litJobs,
                        SeqEnt* __restrict__ seqTabs, SeqJob* __restrict__ seqJobs) {
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    if (ROLE == 0) {
        const uint32_t lane = threadIdx.x & 31u, wib = threadIdx.x >> 5;
        for (uint32_t bi = blockIdx.x * D1_WARPS(0) + wib; bi < nBlocks; bi += gridDim.x * D1_WARPS(0)) {
            const DecBlock blk = blocks[bi];
            if (blk.type != 2) continue;
            const LitHdr lh = parse_lit_hdr(S, blk.srcOff, blk.cSize);
            uint8_t* lit = lits + (size_t)blk.slot * 131072u;
            if (lh.type == 0) { for (uint32_t i = lane; i < lh.regen; i += 32) lit[i] = (uint8_t)S.u8(blk.srcOff + lh.hdr + i); }
            else if (lh.type == 1) { const uint8_t v = (uint8_t)S.u8(blk.srcOff + lh.hdr); for (uint32_t i = lane; i < lh.regen; i += 32) lit[i] = v; }
            if (lane == 0) { LitJob j; j.off = blk.srcOff + lh.hdr; j.size = lh.csize; j.regen = lh.regen; j.streams = lh.type >= 2 ? lh.streams : 0u; j.type = lh.type; litJobs[bi] = j; }
        }
        return;
    }
    const uint32_t maxSymT[3] = { 35, 31, 52 }, maxLogT[3] = { 9, 8, 9 };
    for (uint32_t bi = blockIdx.x * blockDim.x + threadIdx.x; bi < nBlocks; bi += gridDim.x * blockDim.x) {
        const DecBlock blk = blocks[bi];
        if (blk.type != 2) continue;
        uint32_t err = 0;
        const LitHdr lh = parse_lit_hdr(S, blk.srcOff, blk.cSize);
        const uint32_t so = lh.hdr + lh.csize;
        const SeqHdr sh = parse_seq_hdr(S, blk.srcOff + so, blk.cSize - so);
        const uint32_t nbSeq = sh.nbSeq;
        if (nbSeq > B2Z_DEC_MAXSEQ) err = B2Z_DERR_CORRUPT;
        SeqJob job; job.bsOff = 0; job.bsLeft = 0; job.nbSeq = 0; job.litRegen = lh.regen; job.modes = 0; job.pad = 0;
        for (int t = 0; t < 3; t++) { job.desc[t] = 0; job.avail[t] = 0; }
        if (nbSeq && !err) {
            uint64_t bsOff = blk.srcOff + so + sh.hdr; uint32_t bsLeft = blk.cSize - so - sh.hdr;
            int16_t norm[56];
            for (int t = 0; t < 3 && !err; t++) {
                uint64_t d; uint32_t mode, avail;
                const uint32_t ownMode = (sh.modes >> (6 - 2 * t)) & 3u;
                if (ownMode == 3) {
                    if (!locate_seq_table(S, blocks[blk.tblSrc[t]], t, norm, &d, &mode, &avail) || mode == 3) { err = B2Z_DERR_CORRUPT; break; }
                } else { d = bsOff; mode = ownMode; avail = bsLeft; }
                uint32_t used = 0;
                if (mode == 1) { if (avail < 1 || S.u8(d) > maxSymT[t]) err = B2Z_DERR_CORRUPT; else used = 1; }
                else if (mode == 2) { uint32_t ms = maxSymT[t], lg; used = fse_read_ncount(norm, &ms, &lg, S, d, avail, maxLogT[t]); if (!used) err = B2Z_DERR_CORRUPT; }
                job.desc[t] = d; job.avail[t] = avail; job.modes |= mode << (2 * t);
                if (ownMode != 3) { if (used > bsLeft) err = B2Z_DERR_CORRUPT; else { bsOff += used; bsLeft -= used; } }
            }
            if (!err) { job.bsOff = bsOff; job.bsLeft = bsLeft; job.nbSeq = nbSeq; }
        }
        seqJobs[bi] = job;
        blocks[bi].regen = (err || nbSeq) ? 0u : lh.regen; blocks[bi].nbSeq = 0; blocks[bi].litSize = lh.regen;
        if (err) atomicOr(&blocks[bi].status, err);
    }
}

// Literal streams: B2Z_LIT_BLOCKS blocks per CTA, 4 threads per block (one per Huffman stream).  Thread 0 of a block decodes the
// weights, the block's 4 threads fill its 4 KiB table and decode.
#define B2Z_LIT_BLOCKS 16u
__global__ void __launch_bounds__(B2Z_LIT_BLOCKS * 4u)
zstd_dec_lit_streams_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecBlock* __restrict__ blocks, uint32_t nBlocks,
                            uint8_t* __restrict__ lits, const uint16_t* __restrict__ hufTabs, const LitJob* __restrict__ litJobs) {
    B2Z_EXTERN_SMEM(uint16_t, smTab);                                   // [B2Z_LIT_BLOCKS][2048] decoding tables
    __shared__ uint8_t smW[B2Z_LIT_BLOCKS][256];                        // their weights
    __shared__ uint64_t smRing[B2Z_LIT_BLOCKS * 4u][B2Z_BWD_DEPTH];     // each thread's FastBwd words in flight
    const uint32_t j = threadIdx.x >> 2, k = threadIdx.x & 3u, bi = blockIdx.x * B2Z_LIT_BLOCKS + j;
    const uint32_t lead = (threadIdx.x & 31u) & ~3u;                    // lane of the block's thread 0
    uint16_t* tab = smTab + (size_t)j * 2048u;
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    D1_CLOCKS_START();
    LitJob lj; lj.off = 0; lj.size = 0; lj.regen = 0; lj.streams = 0; lj.type = 0;
    if (bi < nBlocks && blocks[bi].type == 2) lj = litJobs[bi];         // (raw / RLE blocks have no job record)
    // ---- the table: weights (thread 0 of the block), then the fill (the block's 4 threads)
    uint32_t tdesc = 0, nw = 0, maxBits = 0, err = 0;
    if (lj.streams && k == 0) {
        const DecBlock sb = blocks[blocks[bi].hufSrc];
        const LitHdr sh = parse_lit_hdr(S, sb.srcOff, sb.cSize);
        const uint32_t u = (sh.ok && sh.type == 2) ? huf_read_weights(smW[j], &nw, &maxBits, S, sb.srcOff + sh.hdr, sh.csize) : 0u;
        if (!u) err = B2Z_DERR_CORRUPT;
        if (lj.type == 2) tdesc = u;
    }
    err = __shfl_sync(B2Z_FULL, err, lead); tdesc = __shfl_sync(B2Z_FULL, tdesc, lead);
    nw = __shfl_sync(B2Z_FULL, nw, lead); maxBits = __shfl_sync(B2Z_FULL, maxBits, lead);
    __syncwarp();                                                       // the weights are visible to the block's threads
    if (lj.streams && !err) huf_fill(tab, smW[j], nw, maxBits, k, 4u);
    __syncwarp();                                                       // the table is complete
    D1_TICK(D1C_TABLE);
    if (!lj.streams) return;
    if (err) { if (k == 0) atomicOr(&blocks[bi].status, err); return; }
    // ---- the streams: one thread each
    uint8_t* lit = lits + (size_t)blocks[bi].slot * 131072u;
    const uint64_t jOff = lj.off + tdesc;
    const uint32_t jSize = tdesc <= lj.size ? lj.size - tdesc : 0xFFFFFFFFu;
    bool ok = true;
    uint64_t off = 0; uint32_t size = 0, cnt = 0; uint8_t* dst = lit;
    if (jSize == 0xFFFFFFFFu) ok = false;
    else if (lj.streams == 1) { if (k) return; off = jOff; size = jSize; cnt = lj.regen; }
    else {
        if (jSize < 6) ok = false;
        else {
            const uint64_t jt = S.le64(jOff);
            const uint32_t s1 = (uint32_t)jt & 0xFFFFu, s2 = (uint32_t)(jt >> 16) & 0xFFFFu, s3 = (uint32_t)(jt >> 32) & 0xFFFFu;
            const uint32_t seg = (lj.regen + 3u) / 4u;
            if (6u + s1 + s2 + s3 > jSize || seg * 3u > lj.regen) ok = false;
            else {
                const uint32_t s4 = jSize - 6u - s1 - s2 - s3;
                const uint32_t so = k == 0 ? 0u : (k == 1 ? s1 : (k == 2 ? s1 + s2 : s1 + s2 + s3));
                size = k == 0 ? s1 : (k == 1 ? s2 : (k == 2 ? s3 : s4));
                cnt = k < 3 ? seg : lj.regen - 3u * seg;
                off = jOff + 6u + so; dst = lit + k * seg;
            }
        }
    }
    if (ok) {
        FastBwd b;
        if (b.init(&S, smRing[threadIdx.x], off, size)) ok = false;
        else {
            const uint32_t mb = maxBits;
            // symbols are gathered eight at a time and stored as one aligned word (head and tail byte by byte): every thread writes its own stream.
            // Inside a word the reloads come before symbols 0 and 4 in every lane: four symbols of <= 11 bits fit the 57 a reload leaves.
            uint32_t i = 0;
            const uint32_t head = (uint32_t)((8u - ((uintptr_t)dst & 7u)) & 7u);
            for (; i < cnt && i < head; i++) {
                if (b.consumed > 64u - 11u) { D1_TICK(D1C_DECODE); b.reload(); D1_TICK(D1C_REFILL); }
                const uint32_t e = tab[(uint32_t)((b.cont << b.consumed) >> (64u - mb))];
                D1_TICK(D1C_DECODE); dst[i] = (uint8_t)e; b.consumed += (e >> 8); D1_TICK(D1C_STORE);
            }
            for (; i + 8u <= cnt; i += 8u) {
                uint64_t acc = 0;
#pragma unroll
                for (uint32_t q = 0; q < 8u; q++) {
                    if ((q & 3u) == 0) { D1_TICK(D1C_DECODE); b.reload(); D1_TICK(D1C_REFILL); }
                    const uint32_t e = tab[(uint32_t)((b.cont << b.consumed) >> (64u - mb))];
                    acc |= (uint64_t)(e & 255u) << (8u * q); b.consumed += (e >> 8);
                }
                D1_TICK(D1C_DECODE); *reinterpret_cast<uint64_t*>(dst + i) = acc; D1_TICK(D1C_STORE);
            }
            for (; i < cnt; i++) {
                if (b.consumed > 64u - 11u) { D1_TICK(D1C_DECODE); b.reload(); D1_TICK(D1C_REFILL); }
                const uint32_t e = tab[(uint32_t)((b.cont << b.consumed) >> (64u - mb))];
                D1_TICK(D1C_DECODE); dst[i] = (uint8_t)e; b.consumed += (e >> 8); D1_TICK(D1C_STORE);
            }
            ok = b.left() == 0;
            b.drain();
        }
    }
    if (!ok) atomicOr(&blocks[bi].status, B2Z_DERR_CORRUPT);
    D1_CLOCKS_FLUSH(0);
}

// Sequence streams: groups of B2Z_SEQ_BLOCKS blocks, one thread per block (the CTA's other threads leave).  The thread builds its
// block's three tables in its 2.5 KiB of shared memory (about 1 % of the block's decode on text) and decodes the bitstream from
// them: the chain of a sequence is shared-memory loads and bit arithmetic, with no global round trip.  17 x 2560 bytes + the symbol
// table are 43.9 KB per CTA: five CTAs (85 chains) per SM of 228 KB, so 32 768 blocks take three waves on 132 SMs.
#define B2Z_SEQ_BLOCKS 17u
__global__ void __launch_bounds__(128)
zstd_dec_seq_streams_kernel(const uint8_t* __restrict__ src, uint64_t srcSize, DecBlock* __restrict__ blocks, uint32_t nBlocks,
                            uint64_t* __restrict__ seqs, const SeqEnt* __restrict__ seqTabs, const SeqJob* __restrict__ seqJobs) {
    __shared__ uint32_t k_seqSym[89];                                   // LL symbols [0,36) | ML symbols [36,89): baseline | extra bits << 24
    __shared__ SeqEnt smTab[B2Z_SEQ_BLOCKS][B2Z_SEQ_TAB];
    __shared__ uint64_t smRing[B2Z_SEQ_BLOCKS][B2Z_BWD_DEPTH];         // each thread's FastBwd words in flight
    for (uint32_t i = threadIdx.x; i < 89u; i += blockDim.x) k_seqSym[i] = i < 36u ? k_LL_base[i] | ((uint32_t)k_LL_bits[i] << 24) : k_ML_base[i - 36u] | ((uint32_t)k_ML_bits[i - 36u] << 24);
    __syncthreads();
    if (threadIdx.x >= B2Z_SEQ_BLOCKS) return;
    SeqEnt* tab = smTab[threadIdx.x];
    Src S; S.w = reinterpret_cast<const uint64_t*>(src); S.nWords = (srcSize + 7) >> 3; S.size = srcSize;
    D1_CLOCKS_START();
    for (uint32_t g = blockIdx.x; (uint64_t)g * B2Z_SEQ_BLOCKS < nBlocks; g += gridDim.x) {
        const uint32_t bi = g * B2Z_SEQ_BLOCKS + threadIdx.x;
        if (bi >= nBlocks) break;
        if (blocks[bi].type != 2) continue;
        const SeqJob j = seqJobs[bi];
        if (!j.nbSeq) continue;
        uint32_t err = 0, logs[3] = { 0, 0, 0 };
        {
            const uint32_t maxSymT[3] = { 35, 31, 52 }, maxLogT[3] = { 9, 8, 9 }, defMax[3] = { 35, 28, 52 }, defLog[3] = { 6, 5, 6 };
            int16_t norm[56];
            for (int t = 0; t < 3 && !err; t++) {
                const uint32_t mode = (j.modes >> (2 * t)) & 3u;
                if (mode == 0) {
                    const int16_t* dn = t == 0 ? k_LL_defNorm : (t == 1 ? k_OF_defNorm : k_ML_defNorm);
                    for (uint32_t s = 0; s <= defMax[t]; s++) norm[s] = dn[s];
                    if (!build_seq_table(tab + seq_tab_off(t), norm, defMax[t], defLog[t])) err = B2Z_DERR_CORRUPT;
                    logs[t] = defLog[t];
                } else if (mode == 1) {
                    tab[seq_tab_off(t)] = (SeqEnt)(S.u8(j.desc[t]) | (1u << 6)); logs[t] = 0;         // one state: no bits, next state 0
                } else {
                    uint32_t ms = maxSymT[t], lg;
                    if (!fse_read_ncount(norm, &ms, &lg, S, j.desc[t], j.avail[t], maxLogT[t]) || !build_seq_table(tab + seq_tab_off(t), norm, ms, lg)) err = B2Z_DERR_CORRUPT;
                    logs[t] = lg;
                }
            }
        }
        D1_TICK(D1C_TABLE);
        uint32_t regen = 0;
        FastBwd b;
        if (err || b.init(&S, smRing[threadIdx.x], j.bsOff, j.bsLeft)) err = B2Z_DERR_CORRUPT;
        else {
            const SeqEnt* tL = tab; const SeqEnt* tO = tab + 512; const SeqEnt* tM = tab + 768;
            const uint32_t gL = logs[0], gO = logs[1], gM = logs[2];
            uint32_t sL = b.read(gL), sO = b.read(gO), sM = b.read(gM);                               // <= 26 bits
            if (b.left() < 0) err = B2Z_DERR_CORRUPT;
            uint64_t* out = seqs + (size_t)blocks[bi].slot * B2Z_DEC_MAXSEQ;
            uint32_t litUsed = 0, total = 0, near = 0;
            // the repcode history as a function of the history before the block (b2z_dec.h DecBlock::repX): slot = value (sym 0) or
            // (initial slot sym - 1) minus value.  ZSTD_decodeSequence's update rules, zstd_decompress_block.c:1290-1312
            uint32_t v0 = 0, v1 = 0, v2 = 0, y0 = 1, y1 = 2, y2 = 3;
            for (uint32_t i = 0; i < j.nbSeq && !err; i++) {
                const uint32_t eL = tL[sL], eO = tO[sO], eM = tM[sM];                                 // symbol | ns << 6
                const uint32_t aO = eO & 63u;
                if (aO > 30u) { err = B2Z_DERR_UNSUPPORTED; break; }
                const uint32_t xL = k_seqSym[eL & 63u], xM = k_seqSym[36u + (eM & 63u)];
                const uint32_t aL = xL >> 24, aM = xM >> 24;
                D1_TICK(D1C_DECODE); b.reload(); D1_TICK(D1C_REFILL);
                const uint32_t ob = (1u << aO) + b.read(aO);
                if (aO + aM + aL > 56u) { D1_TICK(D1C_DECODE); b.reload(); D1_TICK(D1C_REFILL); }
                const uint32_t ml = (xM & 0xFFFFFFu) + b.read(aM);
                const uint32_t ll = (xL & 0xFFFFFFu) + b.read(aL);
                if (i + 1 < j.nbSeq) {
                    if (aO + aM + aL > 30u) { D1_TICK(D1C_DECODE); b.reload(); D1_TICK(D1C_REFILL); }                                                 // + <= 26 state bits
                    const uint32_t nL = eL >> 6, nM = eM >> 6, nO = eO >> 6;
                    const uint32_t bL = gL - highbit32(nL), bM = gM - highbit32(nM), bO = gO - highbit32(nO);
                    sL = ((nL << bL) - (1u << gL)) + b.read(bL); sM = ((nM << bM) - (1u << gM)) + b.read(bM); sO = ((nO << bO) - (1u << gO)) + b.read(bO);
                }
                litUsed += ll; total += ll + ml;
                if (b.left() < 0 || litUsed > j.litRegen || total > 131072u || ob >= (1u << 30)) { err = B2Z_DERR_CORRUPT; break; }
                D1_TICK(D1C_DECODE); out[i] = SEQ_PACK(ob, ll, ml); D1_TICK(D1C_STORE);
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
            b.drain();
            regen = total + (j.litRegen - litUsed);
            if (regen > 131072u) err = B2Z_DERR_CORRUPT;
        }
        D1_TICK(D1C_DECODE);
        blocks[bi].regen = err ? 0u : regen; blocks[bi].nbSeq = err ? 0u : j.nbSeq;
        if (err) atomicOr(&blocks[bi].status, err);
        D1_TICK(D1C_STORE);
    }
    D1_CLOCKS_FLUSH(1);
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
    // scratch layout: litJobs [nBlocks] | seqJobs [nBlocks]; the tables themselves never leave shared memory
    LitJob* litJobs = (LitJob*)scratch;
    SeqJob* seqJobs = (SeqJob*)((uint8_t*)scratch + (size_t)nBlocks * sizeof(LitJob));
    // The literal and the sequence kernels only read src/blocks and write disjoint outputs, so they may run on two streams
    // (stLit != st).  The stream kernels each fill the GPU's shared memory, so co-scheduling them gains nothing;
    // the host dispatcher passes stLit == st.
    if (stLit != st) { cudaEventRecord(evFork, st); cudaStreamWaitEvent(stLit, evFork, 0); }
    const uint32_t cap = smCount * 16u;
    { uint32_t grid = (nBlocks + D1_WARPS(0) - 1) / D1_WARPS(0); if (grid > cap) grid = cap;
      zstd_dec_entropy_kernel<0><<<grid, D1_WARPS(0) * 32, 0, stLit>>>(src, srcSize, blocks, nBlocks, lits, nullptr, litJobs, nullptr, seqJobs);
      cudaFuncSetAttribute(zstd_dec_lit_streams_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(B2Z_LIT_BLOCKS * 4096u));
      cudaFuncSetAttribute(zstd_dec_lit_streams_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
      zstd_dec_lit_streams_kernel<<<(nBlocks + B2Z_LIT_BLOCKS - 1u) / B2Z_LIT_BLOCKS, B2Z_LIT_BLOCKS * 4u, B2Z_LIT_BLOCKS * 4096u, stLit>>>(src, srcSize, blocks, nBlocks, lits, nullptr, litJobs); }
    { const uint32_t threads = D1_WARPS(1) * 32;
      zstd_dec_entropy_kernel<1><<<(nBlocks + threads - 1) / threads, threads, 0, st>>>(src, srcSize, blocks, nBlocks, lits, nullptr, litJobs, nullptr, seqJobs);
      cudaFuncSetAttribute(zstd_dec_seq_streams_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
      zstd_dec_seq_streams_kernel<<<(nBlocks + B2Z_SEQ_BLOCKS - 1u) / B2Z_SEQ_BLOCKS, 32, 0, st>>>(src, srcSize, blocks, nBlocks, seqs, nullptr, seqJobs); }   // one warp: B2Z_SEQ_BLOCKS chains
    if (stLit != st) { cudaEventRecord(evJoin, stLit); cudaStreamWaitEvent(st, evJoin, 0); }
}
#ifdef B2Z_D1_CLOCKS
// the per-phase cycle sums of every stream thread since the last call (literal kernel's D1C_* order, then the sequence kernel's); clears them
extern "C" int b200z_d1_clocks(unsigned long long* out) {
    static const unsigned long long zero[2 * D1C_N] = {};
    cudaError_t e = cudaMemcpyFromSymbol(out, d1_clocks, sizeof(d1_clocks));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(d1_clocks, zero, sizeof(d1_clocks));
    return (int)e;
}
#endif
size_t zstd_dec_entropy_scratch_bytes(uint32_t nBlocks) { return (size_t)nBlocks * (sizeof(LitJob) + sizeof(SeqJob)) + 256u; }
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
