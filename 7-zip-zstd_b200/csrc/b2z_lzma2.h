// b2z_lzma2.h -- LZMA2 (7-Zip method 21) structures and launchers (internal to libb200z.so).
//
// Unit of parallelism = the reference's own: a run of chunks that starts with a dictionary reset
// (control byte 0x01 or >= 0xE0) is decodable on its own -- /root/reference/C/Lzma2DecMt.c:237-414
// (Lzma2DecMt_MtCallback_Parse) cuts streams at exactly these points.
//
// The chunk header format is stated here once: lzma2_chunk reads a header (the walk, the decoder's lane 0, b200z_lzma2_stream_prefix),
// lzma2_chunk_write writes one (both stage R kernels), lzma2_dict_size / lzma2_dict_prop convert the 1-byte coder property.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "b2z_dec.h"

namespace b2z {

// Dictionary size of the 1-byte coder property, dictProp <= 40 (Lzma2Decoder.cpp:40-48 / Lzma2Dec.c:29-31)
__host__ __device__ inline uint32_t lzma2_dict_size(uint32_t dictProp) { return dictProp == 40 ? 0xFFFFFFFFu : ((2u | (dictProp & 1u)) << (dictProp / 2u + 11u)); }
// The property of a 2^frameLog-byte dictionary (Lzma2Enc_WriteProperties, Lzma2Enc.c:671)
__host__ __device__ inline uint32_t lzma2_dict_prop(uint32_t frameLog) { return (frameLog - 12u) * 2u; }

// Whether control byte ctl starts a chunk that resets the dictionary: a stored chunk 0x01 or an LZMA chunk 0xE0-0xFF
__host__ __device__ inline bool lzma2_is_reset(uint32_t ctl) { return ctl == 1u || ctl >= 0xE0u; }

enum : uint32_t { LZ2_CHUNK_END = 0, LZ2_CHUNK_STORED = 1, LZ2_CHUNK_LZMA = 2 };       // Lz2Chunk::kind

struct Lz2Chunk {
    uint32_t status;     // 0, B2Z_DERR_TRUNCATED (the header is cut off) or B2Z_DERR_CORRUPT; the fields below hold only when 0
    uint32_t kind;       // LZ2_CHUNK_*
    bool reset;          // the chunk resets the dictionary
    uint32_t mode;       // LZMA chunk: 0 no reset, 1 state, 2 state + properties, 3 state + properties + dictionary; else 0
    uint32_t hdr;        // header bytes (the end marker: 1)
    uint32_t unpack;     // decoded bytes
    uint32_t pack;       // payload bytes after the header (a stored chunk: unpack)
    uint32_t lc, lp, pb; // from the property byte (mode >= 2); else 0
};

// The chunk header at p, of which avail >= 1 bytes exist (Lzma2Dec.c:97-165, Lzma2Dec_UpdateState).  needInit: the lowest LZMA control
// byte allowed next -- 0xE0 at the start of a stream -- updated for the next header.  A stored chunk is checked for its size before the
// needInit rule, an LZMA chunk after it: a short buffer is truncated or corrupt by that order.
__host__ __device__ inline Lz2Chunk lzma2_chunk(const uint8_t* p, uint64_t avail, uint32_t& needInit) {
    Lz2Chunk c; c.status = 0; c.kind = LZ2_CHUNK_END; c.mode = 0; c.hdr = 1; c.unpack = 0; c.pack = 0; c.lc = 0; c.lp = 0; c.pb = 0;
    const uint32_t ctl = p[0];
    c.reset = lzma2_is_reset(ctl);
    if (ctl == 0) return c;
    if (ctl <= 2) {
        c.kind = LZ2_CHUNK_STORED; c.hdr = 3;
        if (avail < 3) { c.status = B2Z_DERR_TRUNCATED; return c; }
        if (ctl == 1) needInit = 0xC0; else if (needInit == 0xE0) { c.status = B2Z_DERR_CORRUPT; return c; }
        c.unpack = c.pack = (((uint32_t)p[1] << 8) | p[2]) + 1u;
        return c;
    }
    if (ctl < 0x80 || ctl < needInit) { c.status = B2Z_DERR_CORRUPT; return c; }
    needInit = 0;
    c.kind = LZ2_CHUNK_LZMA; c.mode = (ctl >> 5) & 3u; c.hdr = c.mode >= 2 ? 6u : 5u;
    if (avail < c.hdr) { c.status = B2Z_DERR_TRUNCATED; return c; }
    c.unpack = (((ctl & 0x1Fu) << 16) | ((uint32_t)p[1] << 8) | p[2]) + 1u;
    c.pack = (((uint32_t)p[3] << 8) | p[4]) + 1u;
    if (c.mode >= 2) {
        uint32_t d = p[5];
        if (d >= 225) { c.status = B2Z_DERR_CORRUPT; return c; }
        c.lc = d % 9u; d /= 9u; c.lp = d % 5u; c.pb = d / 5u;
        if (c.lc + c.lp > 4) c.status = B2Z_DERR_CORRUPT;
    }
    return c;
}

struct Lz2Block {
    uint64_t srcOff;     // first chunk header of the block
    uint64_t srcEnd;     // offset of the next block's first chunk header (or of the end marker)
    uint64_t dstOff;     // output offset
    uint64_t dstSize;    // sum of the block's chunk unpack sizes
};

struct Lz2Counts {
    uint32_t nBlocks;    // blocks found (may exceed the capacity given to the walk: caller re-runs)
    uint32_t status;     // B2Z_DERR_* bits
    uint32_t maxLcLp;    // largest lc+lp of any property byte in the stream (sizes the literal model)
    uint32_t pad;
    uint64_t srcUsed;    // bytes up to and including the end marker
    uint64_t total;      // decoded size
};

// Chunk-header walk shared by the device pre-pass and the host-side stream_info (headers only, no payload access): cuts the stream
// at its dictionary resets and emits one Lz2Block each.
template <class Emit>
__host__ __device__ inline void lzma2_walk(const uint8_t* src, uint64_t srcSize, Lz2Counts& c, Emit emit) {
    uint64_t ip = 0, total = 0, blkSrc = 0, blkDst = 0;
    uint32_t nb = 0, status = 0, maxLcLp = 0, needInit = 0xE0;
    bool ended = false;
    while (ip < srcSize) {
        const Lz2Chunk ch = lzma2_chunk(src + ip, srcSize - ip, needInit);
        if (ch.status) break;                       // corrupt or cut off: no end marker (status bit 0 below)
        if (ch.kind == LZ2_CHUNK_END) { ip++; ended = true; break; }
        if (ch.lc + ch.lp > maxLcLp) maxLcLp = ch.lc + ch.lp;
        if (ch.hdr + ch.pack > srcSize - ip) break;
        if (ch.reset) {
            if (nb) emit(nb - 1, blkSrc, ip, blkDst, total - blkDst);
            nb++; blkSrc = ip; blkDst = total;
        }
        total += ch.unpack; ip += ch.hdr + ch.pack;
        if (total - blkDst > 0xFFFFFFFFull) { status |= 2u; break; }     // one block >= 4 GiB: positions are 32-bit here
    }
    if (!ended) status |= 1u;                       // corrupt, truncated or no end marker
    if (nb) emit(nb - 1, blkSrc, ended ? ip - 1 : ip, blkDst, total - blkDst);
    c.nBlocks = nb; c.status = status; c.maxLcLp = maxLcLp; c.pad = 0; c.srcUsed = ip; c.total = total;
}

// probability model layout shared by decoder and encoder (uint16 probabilities; own layout, same sets as LzmaDec.c:130-227)
enum : uint32_t {
    P_ISMATCH = 0,                    // [12][16]
    P_ISREP = 192,                    // [12]
    P_ISREPG0 = 204, P_ISREPG1 = 216, P_ISREPG2 = 228,
    P_ISREP0LONG = 240,               // [12][16]
    P_POSSLOT = 432,                  // [4][64]
    P_SPECPOS = 688,                  // [115] (+1 pad)
    P_ALIGN = 804,                    // [16]
    P_LEN = 820,                      // choice, choice2, low[16][8], mid[16][8], high[256]  = 514
    P_REPLEN = 1334,
    P_LIT = 1848,                     // [0x300 << (lc+lp)]
    L_CHOICE = 0, L_CHOICE2 = 1, L_LOW = 2, L_MID = 130, L_HIGH = 258
};

// ---- encoder (stage R): one thread per frame turns the stage-M sequences into one dictionary-reset LZMA2 block in its slot

// Closes a chunk of a stage R slot (Lzma2Enc.c:183-238): out[chunkOut, op) holds hdr free header bytes, then the range-coded ones; s: its
// unpack input bytes.  Writes the LZMA chunk header, or rewrites the chunk as a stored one (op moves) when coding did not save 3 bytes.
// needDict / needProps / needState say what the chunk resets and are updated for the next chunk.
__device__ inline void lzma2_chunk_write(uint8_t* out, uint32_t& op, uint32_t chunkOut, uint32_t hdr, const uint8_t* s, uint32_t unpack,
                                         uint32_t props, bool& needDict, bool& needProps, bool& needState) {
    const uint32_t pack = op - chunkOut - hdr;
    uint8_t* h = out + chunkOut;
    if (pack + 2u >= unpack) {
        h[0] = needDict ? 1 : 2; h[1] = (uint8_t)((unpack - 1u) >> 8); h[2] = (uint8_t)(unpack - 1u);
        for (uint32_t i = 0; i < unpack; i++) h[3u + i] = __ldg(s + i);
        op = chunkOut + 3u + unpack;
        needDict = false; needState = true;
        return;
    }
    const uint32_t mode = needDict ? 3u : (needProps ? 2u : (needState ? 1u : 0u));
    h[0] = (uint8_t)(0x80u | (mode << 5) | ((unpack - 1u) >> 16)); h[1] = (uint8_t)((unpack - 1u) >> 8); h[2] = (uint8_t)(unpack - 1u);
    h[3] = (uint8_t)((pack - 1u) >> 8); h[4] = (uint8_t)(pack - 1u);
    if (mode >= 2u) h[5] = (uint8_t)props;
    needDict = needProps = needState = false;
}

struct EncGeom;
size_t lzma2_enc_slot_stride(const EncGeom& g);
uint32_t lzma2_enc_slices_per_frame(const EncGeom& g);
size_t lzma2_enc_model_bytes(uint32_t nChains, uint32_t flags = 0);   // mode 3 (32 chains per warp): the chains' models, passed as litSpill
uint32_t lzma2_enc_smem_chains_per_sm(uint32_t flags);     // chains per SM with the whole model in shared memory (modes 0 / 1)
cudaError_t launch_lzma2_enc_range(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint64_t* seqs, const uint32_t* nseq,
                                   uint8_t* slots, uint32_t* slotSize, uint32_t nFrames, uint16_t* litSpill, uint32_t smCount, int mode,
                                   uint32_t* status, cudaStream_t st);
// offsets (one CTA scan) + gather of the frame slots into the contiguous chunk stream, end marker appended
void launch_lzma2_enc_assemble(const uint8_t* slots, const uint32_t* slotSize, uint32_t nPieces, uint32_t slotStride, uint64_t* pieceOff,
                               uint8_t* dst, uint64_t* outSize, cudaStream_t st);

// ---- encoder, price-based parse (lzma2_parse.cu): stage C (candidates, one warp per frame; nWarps table sets) and stage P
// (dynamic programme, one warp per state-reset slice) fill the per-block sequence arrays stage R reads
size_t lzma2_cand_table_bytes(const EncGeom& g, uint32_t nWarps);
size_t lzma2_parse_smem_bytes(uint32_t flags = 0);       // one warp's working set: grows with lc + lp (flags bits 15-23)
void launch_lzma2_cand(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t* tables, uint32_t nWarps, uint32_t* cand /* [srcSize * 4] */, cudaStream_t st);
cudaError_t launch_lzma2_parse(const uint8_t* src, uint64_t srcSize, const EncGeom& g, const uint32_t* cand, uint64_t* seqs,
                               uint32_t* nseq /* one counter per 128 KiB block, zeroed here */, cudaStream_t st);

void launch_lzma2_walk(const uint8_t* src, uint64_t srcSize, Lz2Block* blocks, uint32_t cap, Lz2Counts* counts, cudaStream_t st);
// one warp per block; returns cudaError of the launch configuration (shared memory opt-in)
size_t lzma2_lit_spill_bytes(uint32_t nBlocks, uint32_t maxLcLp);
cudaError_t launch_lzma2_decode(const uint8_t* src, const Lz2Block* blocks, uint32_t nBlocks, uint32_t maxLcLp, uint32_t dictSize,
                                uint8_t* dst, Lz2Counts* counts, uint16_t* litSpill, uint32_t smCount, int mode, cudaStream_t st);

}  // namespace b2z
