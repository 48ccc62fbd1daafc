// b2z_lzma2.h -- LZMA2 (7-Zip method 21) structures and launchers (internal to libb200z.so).
//
// Unit of parallelism = the reference's own: a run of chunks that starts with a dictionary reset
// (control byte 0x01 or >= 0xE0) is decodable on its own -- /root/reference/C/Lzma2DecMt.c:237-414
// (Lzma2DecMt_MtCallback_Parse) cuts streams at exactly these points.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2z {

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

// Chunk-header walk shared by the device pre-pass and the host-side stream_info (headers only, no payload access).
// Lzma2Dec.c:97-165 (Lzma2Dec_UpdateState): control byte, 2+2 size bytes, optional property byte, needInitLevel rule.
template <class Emit>
__host__ __device__ inline void lzma2_walk(const uint8_t* src, uint64_t srcSize, Lz2Counts& c, Emit emit) {
    uint64_t ip = 0, total = 0, blkSrc = 0, blkDst = 0;
    uint32_t nb = 0, status = 0, maxLcLp = 0, needInit = 0xE0;
    bool ended = false;
    while (ip < srcSize) {
        const uint32_t ctl = src[ip];
        if (ctl == 0) { ip++; ended = true; break; }
        uint64_t hdr, pack, unpack; bool reset;
        if (ctl <= 2) {
            if (ip + 3 > srcSize) break;
            hdr = 3; pack = unpack = (((uint64_t)src[ip + 1] << 8) | src[ip + 2]) + 1; reset = ctl == 1;
            if (ctl == 1) needInit = 0xC0; else if (needInit == 0xE0) { status |= 1u; break; }
        } else {
            if (ctl < 0x80 || ctl < needInit) { status |= 1u; break; }
            needInit = 0;
            const uint32_t mode = (ctl >> 5) & 3u;
            hdr = 5 + (mode >= 2 ? 1 : 0);
            if (ip + hdr > srcSize) break;
            unpack = ((((uint64_t)ctl & 0x1F) << 16) | ((uint64_t)src[ip + 1] << 8) | src[ip + 2]) + 1;
            pack = (((uint64_t)src[ip + 3] << 8) | src[ip + 4]) + 1;
            reset = mode == 3;
            if (mode >= 2) {
                uint32_t d = src[ip + 5];
                if (d >= 225) { status |= 1u; break; }
                const uint32_t lc = d % 9; d /= 9; const uint32_t lp = d % 5;
                if (lc + lp > 4) { status |= 1u; break; }
                if (lc + lp > maxLcLp) maxLcLp = lc + lp;
            }
        }
        if (ip + hdr + pack > srcSize) break;
        if (reset) {
            if (nb) emit(nb - 1, blkSrc, ip, blkDst, total - blkDst);
            nb++; blkSrc = ip; blkDst = total;
        }
        total += unpack; ip += hdr + pack;
        if (total - blkDst > 0xFFFFFFFFull) { status |= 2u; break; }     // one block >= 4 GiB: positions are 32-bit here
    }
    if (!ended) status |= 1u;                       // truncated / no end marker
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
