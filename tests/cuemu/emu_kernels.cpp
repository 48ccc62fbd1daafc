// emu_kernels.cpp -- TEST INFRASTRUCTURE ONLY: the kernel SOURCES of 7-zip-zstd_b200/csrc compiled for the host through
// tests/cuemu/cuemu.h (see there), with C entry points the CPU tests call.  Built by tests/cuemu/Makefile into
// tests/cuemu/libcuemu_kernels.so; never part of libb200z.so.
#define B2Z_CUEMU 1
#include "cuemu.h"
#include "../../7-zip-zstd_b200/csrc/zstd_enc_find.cu"
#include "../../7-zip-zstd_b200/csrc/zstd_enc_dp.cu"
#include "../../7-zip-zstd_b200/csrc/zstd_enc_ldm.cu"
#include "../../7-zip-zstd_b200/csrc/lzma2_parse.cu"
#include "../../7-zip-zstd_b200/csrc/zstd_enc_parse.cu"
#include "../../7-zip-zstd_b200/csrc/zstd_enc_entropy.cu"
#include "../../7-zip-zstd_b200/csrc/zstd_enc_frame.cu"
#include "../../7-zip-zstd_b200/csrc/b2z_crc.cu"
#include "../../7-zip-zstd_b200/csrc/b2z_filter.cu"
#include "../../7-zip-zstd_b200/csrc/lzma2_enc.cu"
#include "../../7-zip-zstd_b200/csrc/lzma2_dec.cu"
#include "../../7-zip-zstd_b200/csrc/zstd_dec.cu"

using namespace b2z;

static EncGeom geom(uint32_t frameLog, uint32_t windowLog, uint32_t chunkLog, uint32_t flags) {
    EncGeom g; memset(&g, 0, sizeof(g));
    g.frameLog = frameLog; g.hashLogL = B2Z_DEF_HASHLOG_L; g.hashLogS = (flags & B2Z_FLAG_FIND_FAST) ? B2Z_DEF_HASHLOG_L : B2Z_DEF_HASHLOG_S; g.windowLog = windowLog; g.flags = flags; g.chunkLog = chunkLog; g.frameSizes = nullptr;
    return g;
}

extern "C" {

// stage F (zstd_enc_find_kernel): candidate words, frames back to back; nCtas CTAs loop over the frames
static uint64_t run_find(const uint8_t* src, uint64_t srcSize, const EncGeom& g, uint32_t nCtas, uint32_t* cand) {
    const size_t smem = (((g.flags & B2Z_FLAG_FIND_FAST) ? 0 : ((size_t)1 << g.hashLogL)) + ((size_t)1 << g.hashLogS) + 1024u) * 4u;
    uint32_t err = 0;
    const int mode = (g.flags & B2Z_FLAG_FIND_FAST) ? 1 : ((g.flags & B2Z_FLAG_FIND_STEP) ? 2 : 0);
#define EMU_FIND(WPG, G) (mode == 1 ? cuemu::launch(dim3(nCtas), dim3(WPG * G * 32), smem, [&] { zstd_enc_find_kernel<WPG, G, 1>(src, srcSize, g, cand, nullptr, 0, &err); }) \
                        : mode == 2 ? cuemu::launch(dim3(nCtas), dim3(WPG * G * 32), smem, [&] { zstd_enc_find_kernel<WPG, G, 2>(src, srcSize, g, cand, nullptr, 0, &err); }) \
                                    : cuemu::launch(dim3(nCtas), dim3(WPG * G * 32), smem, [&] { zstd_enc_find_kernel<WPG, G, 0>(src, srcSize, g, cand, nullptr, 0, &err); }))
    switch (g.chunkLog) {
    case 5: return EMU_FIND(1, 7);
    case 6: return EMU_FIND(2, 7);
    case 7: return EMU_FIND(4, 7);
    case 8: return EMU_FIND(8, 4);
    }
#undef EMU_FIND
    return 0;
}
uint64_t emu_zstd_enc_find(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t windowLog, uint32_t chunkLog, uint32_t flags, uint32_t nCtas, uint32_t* cand) {
    return run_find(src, srcSize, geom(frameLog, windowLog, chunkLog, flags), nCtas, cand);
}

// long mode: stage F per region, then stage L per frame (zstd_enc_ldm_kernel): candidate words as the oracle's b2zo_zstd_candidates
uint64_t emu_zstd_enc_find_long(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t windowLog, uint32_t regionLog, uint32_t ldmLog, uint32_t nCtas, uint32_t* cand) {
    EncGeom g = geom(frameLog, windowLog, B2Z_DEF_CHUNKLOG, 0); g.regionLog = regionLog; g.ldmLog = ldmLog;
    EncGeom gF = g; gF.frameLog = regionLog;
    uint64_t c = run_find(src, srcSize, gF, nCtas, cand);
    const uint32_t E = B2Z_LDM_EPOCHLOG(windowLog);
    std::vector<uint32_t> tables((size_t)((srcSize + (1ull << E) - 1) >> E) << ldmLog, 0xFFFFFFFFu);   // (launch_zstd_enc_ldm: cudaMemsetAsync 0xFF)
    c += cuemu::launch(dim3(nCtas), dim3(B2Z_LDM_THREADS), 0, [&] { zstd_enc_ldm_kernel<0>(src, srcSize, g, cand, tables.data()); });
    c += cuemu::launch(dim3(nCtas), dim3(B2Z_LDM_THREADS), 0, [&] { zstd_enc_ldm_kernel<1>(src, srcSize, g, cand, tables.data()); });
    return c;
}

// stage F + stage G (zstd_enc_find_kernel, zstd_enc_dp_kernel): per-block sequences and literals as the oracle's b2zo_zstd_find_sequences
uint64_t emu_zstd_enc_match(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t windowLog, uint32_t chunkLog, uint32_t flags, uint32_t nCtas,
                            uint64_t* seqs, uint32_t* nseq, uint8_t* lits, uint32_t* nlit) {
    const EncGeom g = geom(frameLog, windowLog, chunkLog, flags);
    const uint64_t F = 1ull << frameLog, nFrames = (srcSize + F - 1) >> frameLog;
    std::vector<uint32_t> cand((size_t)nFrames * F + 16, 0xCDCDCDCDu);
    std::vector<uint8_t> choice((size_t)nFrames * F + 16, 0xCD);
    uint64_t c = run_find(src, srcSize, g, nCtas, cand.data());
    const uint32_t nBlockSlots = (uint32_t)(nFrames << (frameLog - 17u));
    c += cuemu::launch(dim3((nBlockSlots + B2Z_DP_WARPS - 1) / B2Z_DP_WARPS), dim3(B2Z_DP_WARPS * 32), sizeof(DpWarpSmem) * B2Z_DP_WARPS, [&] {
        zstd_enc_dp_kernel(src, srcSize, g, cand.data(), choice.data(), seqs, nseq, lits, nlit, nBlockSlots);
    });
    return c;
}

// stage C (lzma2_cand_kernel)
uint64_t emu_lzma2_cand(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, uint32_t nWarps, uint32_t* cand) {
    const EncGeom g = geom(frameLog, frameLog, B2Z_DEF_CHUNKLOG, flags);
    std::vector<uint32_t> tables((size_t)nWarps * lzma2_cand_table_words(frameLog), 0xCDCDCDCDu);
    return cuemu::launch(dim3(nWarps), dim3(32), 0, [&] { lzma2_cand_kernel(src, srcSize, g, tables.data(), cand); });
}

// stage P (lzma2_parse_kernel); nseq is zeroed here as launch_lzma2_parse does
uint64_t emu_lzma2_parse(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, const uint32_t* cand, uint64_t* seqs, uint32_t* nseq) {
    const EncGeom g = geom(frameLog, frameLog, B2Z_DEF_CHUNKLOG, flags);
    const uint64_t F = 1ull << frameLog;
    const uint32_t nFrames = (uint32_t)((srcSize + F - 1) >> frameLog), bpf = (uint32_t)(F >> 17);
    const uint32_t spf = bpf / B2Z_LZ2_SLICE_BLOCKS(frameLog, flags), nChains = nFrames * spf;
    memset(nseq, 0, (size_t)nFrames * bpf * sizeof(uint32_t));
    return cuemu::launch(dim3(nChains), dim3(32), lzma2_parse_smem_bytes(), [&] { lzma2_parse_kernel(src, srcSize, g, cand, seqs, nseq, nChains); });
}

// stage Z (zstd_enc_parse_kernel)
uint64_t emu_zstd_enc_parse(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, const uint32_t* cand,
                            uint64_t* seqs, uint32_t* nseq, uint8_t* lits, uint32_t* nlit) {
    const EncGeom g = geom(frameLog, frameLog, B2Z_DEF_CHUNKLOG, flags);
    const uint64_t F = 1ull << frameLog;
    const uint32_t nFrames = (uint32_t)((srcSize + F - 1) >> frameLog);
    const uint32_t nBlocks = (nFrames - 1u) * (uint32_t)(F >> 17) + (uint32_t)((srcSize - (uint64_t)(nFrames - 1u) * F + B2Z_BLOCK - 1u) / B2Z_BLOCK);
    return cuemu::launch(dim3(nBlocks), dim3(32), zstd_enc_parse_smem_bytes(), [&] { zstd_enc_parse_kernel(src, srcSize, g, cand, seqs, nseq, lits, nlit, nBlocks); });
}

// stage E (zstd_enc_entropy_kernel): per-block compressed bodies in slots of B2Z_SLOT bytes.  GPU-verified on stage M's sequences;
// here it is also fed stage Z's
uint64_t emu_zstd_enc_entropy(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, const uint64_t* seqs, const uint32_t* nseq,
                              const uint8_t* lits, const uint32_t* nlit, uint8_t* slots, uint32_t* slotSize, uint32_t nBlocks) {
    const EncGeom g = geom(frameLog, frameLog, B2Z_DEF_CHUNKLOG, flags);
    return cuemu::launch(dim3((nBlocks + B2Z_ENT_WARPS - 1) / B2Z_ENT_WARPS), dim3(B2Z_ENT_WARPS * 32), 0,
                         [&] { zstd_enc_entropy_kernel(src, srcSize, g, seqs, nseq, lits, nlit, slots, slotSize, nBlocks); });
}
uint32_t emu_slot_bytes() { return B2Z_SLOT; }

// crc_pieces_kernel: per-piece CRC32 / CRC64 (pieces of 2^pieceLog bytes, or the given ranges)
uint64_t emu_crc_pieces(const uint8_t* src, uint64_t n, uint32_t pieceLog, const uint64_t* off, const uint64_t* len, uint32_t nPieces, uint32_t width, void* out) {
    const dim3 grid((nPieces + 127u) / 128u), block(128);
    if (width == 32) return cuemu::launch(grid, block, 0, [&] { crc_pieces_kernel<uint32_t>(src, n, pieceLog, off, len, nPieces, B2Z_CRC32_POLY, (uint32_t*)out); });
    return cuemu::launch(grid, block, 0, [&] { crc_pieces_kernel<uint64_t>(src, n, pieceLog, off, len, nPieces, B2Z_CRC64_POLY, (uint64_t*)out); });
}

// filters (b2z_filter.cu), in place on `data`; same launch shapes as b200z_filter_device
void emu_filter(uint32_t methodId, int enc, uint8_t* data, uint64_t n, uint32_t prop, uint32_t unitLog) {
    if (methodId == B200Z_F_DELTA) {
        if (enc) {
            std::vector<uint8_t> copy(data, data + n);
            cuemu::launch(dim3((uint32_t)((n + 255) / 256 < 64 ? (n + 255) / 256 : 64)), dim3(256), 0, [&] { delta_enc_kernel(copy.data(), data, n, prop, unitLog); });
        } else {
            const uint32_t rows = (65536u / prop) ? (65536u / prop) : 1u;
            const uint64_t tileBytes = (uint64_t)rows * prop;
            const uint32_t tiles = (uint32_t)((n + tileBytes - 1) / tileBytes);
            std::vector<uint8_t> sums((size_t)tiles * prop + 64, 0xCD);
            cuemu::launch(dim3(tiles), dim3(256), 0, [&] { delta_colsum_kernel(data, n, prop, rows, sums.data()); });
            cuemu::launch(dim3(1), dim3(256), 0, [&] { delta_scan_kernel(sums.data(), tiles, prop); });
            cuemu::launch(dim3(tiles), dim3(256), 0, [&] { delta_dec_kernel(data, n, prop, rows, sums.data()); });
        }
    } else if (methodId == B200Z_F_ARMT) {
        const uint64_t nHalf = n >> 1;
        if (nHalf >= 2) {
            std::vector<uint8_t> copy(data, data + n);
            cuemu::launch(dim3((uint32_t)((nHalf + 255) / 256 < 32 ? (nHalf + 255) / 256 : 32)), dim3(256), 0, [&] { armt_kernel((const uint16_t*)copy.data(), (uint16_t*)data, nHalf, enc, prop, unitLog); });
        }
    } else if (methodId == B200Z_F_X86) {
        if (n >= 5) {
            std::vector<uint8_t> copy(data, data + n);
            const uint64_t threads = (n + 31) / 32;
            cuemu::launch(dim3((uint32_t)((threads + 127) / 128)), dim3(128), 0, [&] { x86_kernel(copy.data(), data, n, prop, enc, unitLog); });
        }
    } else {
        const uint64_t nWords = n >> 2;
        if (nWords) cuemu::launch(dim3((uint32_t)((nWords + 255) / 256 < 32 ? (nWords + 255) / 256 : 32)), dim3(256), 0, [&] { bra_kernel((uint32_t*)data, nWords, methodId, enc, prop, unitLog); });
    }
}

// stage R (lzma2_enc_range_kernel, model in shared memory) + assembly: sequences -> the frame-ordered chunk stream with its end marker
int64_t emu_lzma2_range_and_assemble(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, const uint64_t* seqs, const uint32_t* nseq,
                                     uint8_t* dst, uint64_t dstCap, int glit) {
    const EncGeom g = geom(frameLog, frameLog, B2Z_DEF_CHUNKLOG, flags);
    const uint32_t nFrames = (uint32_t)((srcSize + (1ull << frameLog) - 1) >> frameLog);
    const uint32_t nChains = nFrames * lzma2_enc_slices_per_frame(g);
    const uint32_t stride = (uint32_t)lzma2_enc_slot_stride(g);
    constexpr uint32_t LITN = 0x300u << (B2Z_LZ2_LC + B2Z_LZ2_LP);
    std::vector<uint8_t> slots((size_t)nChains * stride, 0xCD); std::vector<uint32_t> slotSize(nChains + 1, 0xCDCDCDCDu); uint32_t status = 0;
    std::vector<uint16_t> spill(glit == 1 ? (size_t)nChains * LITN : 1);
    std::vector<uint16_t> models(glit == 2 ? lzma2_enc_model_bytes(nChains) / 2 : 1, 0xCDCD);
    if (glit == 2) cuemu::launch(dim3(((nChains + 31u) / 32u + B2Z_R32_WARPS - 1u) / B2Z_R32_WARPS), dim3(32 * B2Z_R32_WARPS), B2Z_R32_WARPS * B2Z_R32_QCAP * 32u * sizeof(uint16_t), [&] {
        lzma2_enc_range32_kernel(src, srcSize, g, seqs, nseq, slots.data(), stride, slotSize.data(), models.data(), &status, nChains); });
    else if (glit) cuemu::launch(dim3((nChains + 1u) / 2u), dim3(64), 2u * P_LIT * sizeof(uint16_t), [&] {
        lzma2_enc_range_kernel<true, 1>(src, srcSize, g, seqs, nseq, slots.data(), stride, slotSize.data(), spill.data(), &status, nChains); });
    else cuemu::launch(dim3(nChains), dim3(32), ((size_t)P_LIT + LITN) * sizeof(uint16_t), [&] {
        lzma2_enc_range_kernel<false, 1>(src, srcSize, g, seqs, nseq, slots.data(), stride, slotSize.data(), nullptr, &status, nChains); });
    if (status) return -1;
    std::vector<uint64_t> off(nChains + 2); uint64_t outSize = 0;
    cuemu::launch(dim3(1), dim3(1024), 0, [&] { lzma2_enc_offsets_kernel(slotSize.data(), nChains, off.data(), &outSize); });
    if (outSize > dstCap) return -2;
    cuemu::launch(dim3(nChains, 4), dim3(256), 0, [&] { lzma2_enc_gather_kernel(slots.data(), stride, slotSize.data(), off.data(), nChains, dst); });
    return (int64_t)outSize;
}

// LZMA2 decoder (lzma2_walk_kernel + lzma2_decode_kernel): chunk stream -> bytes; returns the decoded size or -(status)
int64_t emu_lzma2_decode(const uint8_t* src, uint64_t srcSize, uint32_t dictProp, uint8_t* dst, uint64_t dstCap, int glit) {
    Lz2Counts counts; std::vector<Lz2Block> blocks(srcSize / 8 + 16);
    cuemu::launch(dim3(1), dim3(32), 0, [&] { lzma2_walk_kernel(src, srcSize, blocks.data(), (uint32_t)blocks.size(), &counts); });
    if (counts.status) return -(int64_t)counts.status;
    if (counts.total > dstCap) return -100;
    const uint32_t dictSize = lzma2_dict_size(dictProp);
    const uint32_t litCount = 0x300u << counts.maxLcLp;
    std::vector<uint16_t> spill(glit ? (size_t)counts.nBlocks * litCount : 1);
    if (counts.nBlocks) {
        if (glit) cuemu::launch(dim3(counts.nBlocks), dim3(32), P_LIT * sizeof(uint16_t), [&] { lzma2_decode_kernel<true>(src, blocks.data(), dst, dictSize, &counts, spill.data(), litCount); });
        else cuemu::launch(dim3(counts.nBlocks), dim3(32), ((size_t)P_LIT + litCount) * sizeof(uint16_t), [&] { lzma2_decode_kernel<false>(src, blocks.data(), dst, dictSize, &counts, nullptr, 0); });
    }
    return counts.status ? -(int64_t)counts.status : (int64_t)counts.total;
}

// frame assembly (zstd_enc_checksum / offsets / gather kernels): stage E's slots -> the frames, as launch_zstd_enc_assemble runs them
int64_t emu_zstd_enc_assemble(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, const uint8_t* slots, const uint32_t* slotSize,
                              uint32_t nBlocks, uint8_t* dst, uint64_t dstCap) {
    const EncGeom g = geom(frameLog, frameLog, B2Z_DEF_CHUNKLOG, flags);
    const uint32_t nFrames = (uint32_t)((srcSize + (1ull << frameLog) - 1) >> frameLog);
    std::vector<uint64_t> blockOff(nBlocks + 2), frameOff(nFrames + 2); std::vector<uint32_t> cks(nFrames + 2, 0xCDCDCDCDu); uint64_t outSize = 0;
    if (flags & 2u) cuemu::launch(dim3((nFrames + 63) / 64), dim3(64), 0, [&] { zstd_enc_checksum_kernel(src, srcSize, g, cks.data(), nFrames); });
    cuemu::launch(dim3(1), dim3(1024), 0, [&] { zstd_enc_offsets_kernel(srcSize, g, slotSize, nBlocks, blockOff.data(), &outSize, frameOff.data()); });
    if (outSize > dstCap) return -2;
    cuemu::launch(dim3(nBlocks), dim3(256), 0, [&] { zstd_enc_gather_kernel(srcSize, g, slots, slotSize, blockOff.data(), nBlocks, dst, cks.data()); });
    return (int64_t)outSize;
}

// Zstandard decoder: the kernels in the order and shapes of dec_impl (zstd_dec_api.cu) / the launch_zstd_dec_* functions.
// Returns the decoded size or -(status bits).
static uint32_t g_emu_jump_seglog = B2Z_DEC_JUMP_SEGLOG;                                   // stage J segment size (tests shrink it)
void emu_set_jump_seglog(uint32_t v) { g_emu_jump_seglog = v; }
static int64_t emu_zstd_decode_mode(const uint8_t* src, uint64_t srcSize, uint8_t* dst, uint64_t dstCap, uint32_t jumpMode, uint32_t* nJumpOut);
int64_t emu_zstd_decode(const uint8_t* src, uint64_t srcSize, uint8_t* dst, uint64_t dstCap) { return emu_zstd_decode_mode(src, srcSize, dst, dstCap, 1u, nullptr); }
// jumpMode as B200Z_P_DEC_JUMP; *nJump = frames that went through stage J
int64_t emu_zstd_decode_jump(const uint8_t* src, uint64_t srcSize, uint8_t* dst, uint64_t dstCap, uint32_t jumpMode, uint32_t* nJump) {
    return emu_zstd_decode_mode(src, srcSize, dst, dstCap, jumpMode, nJump);
}
static int64_t emu_zstd_decode_mode(const uint8_t* src, uint64_t srcSize, uint8_t* dst, uint64_t dstCap, uint32_t jumpMode, uint32_t* nJumpOut) {
    if (nJumpOut) *nJumpOut = 0;
    if (!srcSize) return 0;
    uint64_t frameCap = srcSize / 9 + 2, blockCap = srcSize / 3 + 2;
    { const uint64_t lim = srcSize / 128 + 65536; if (blockCap > lim) blockCap = lim; }                  // (the product adds 2^20: table entries only)
    std::vector<DecFrame> frames(frameCap); std::vector<DecBlock> blocks(blockCap);
    DecCounts counts; memset(&counts, 0, sizeof(counts)); uint64_t total = 0;
    uint32_t nFrames = 0;
    for (int pass = 0; pass < 2; pass++) {                                               // dec_impl: size hints trusted first, walked again if that fails
        memset(&counts, 0, sizeof(counts));
        cuemu::launch(dim3(1), dim3(32), 0, [&] { zstd_dec_find_frames_kernel(src, srcSize, frames.data(), (uint32_t)frameCap, &counts, pass == 0 ? 1u : 0u); });
        const uint32_t hinted = counts.nUnits;
        nFrames = counts.nFrames;
        const uint32_t g0 = (nFrames + 63) / 64;
        if (!counts.status && g0) {
            cuemu::launch(dim3(g0), dim3(64), 0, [&] { zstd_dec_count_blocks_kernel(src, srcSize, frames.data(), nFrames, &counts); });
            cuemu::launch(dim3(1), dim3(32), 0, [&] { zstd_dec_scan_blocks_kernel(frames.data(), nFrames, (uint32_t)blockCap, &counts); });
            cuemu::launch(dim3(g0), dim3(64), 0, [&] { zstd_dec_fill_blocks_kernel(src, srcSize, frames.data(), nFrames, blocks.data(), (uint32_t)blockCap, &counts); });
        }
        if (!counts.status || !hinted || (counts.status & ~B2Z_DERR_CORRUPT)) break;
    }
    if (counts.status) return -(int64_t)counts.status;
    const uint32_t nBlocks = counts.nBlocks;
    const uint32_t nSlots = counts.nSlots;                                               // compressed blocks: the only ones with literal / sequence scratch
    std::vector<uint8_t> lits((size_t)nSlots * 131072ull + 64); std::vector<uint64_t> seqs((size_t)nSlots * B2Z_DEC_MAXSEQ + 8);
    std::vector<uint8_t> scratch((size_t)nBlocks * (4096u + 1280u * sizeof(SeqEnt) + sizeof(LitJob) + sizeof(SeqJob)) + 256u, 0xCD);
    if (nBlocks) {
        uint8_t* p = scratch.data();
        uint16_t* hufTabs = (uint16_t*)p; p += (size_t)nBlocks * 4096u;
        SeqEnt* seqTabs = (SeqEnt*)p; p += (size_t)nBlocks * 1280u * sizeof(SeqEnt);
        LitJob* litJobs = (LitJob*)p; p += (size_t)nBlocks * sizeof(LitJob);
        SeqJob* seqJobs = (SeqJob*)p;
        cuemu::launch(dim3((nBlocks + D1_WARPS(0) - 1) / D1_WARPS(0)), dim3(D1_WARPS(0) * 32), 0, [&] { zstd_dec_entropy_kernel<0>(src, srcSize, blocks.data(), nBlocks, lits.data(), hufTabs, litJobs, seqTabs, seqJobs); });
        cuemu::launch(dim3((nBlocks + B2Z_LIT_BLOCKS - 1u) / B2Z_LIT_BLOCKS), dim3(B2Z_LIT_BLOCKS * 4u), B2Z_LIT_BLOCKS * 4096u, [&] { zstd_dec_lit_streams_kernel(src, srcSize, blocks.data(), nBlocks, lits.data(), hufTabs, litJobs); });
        cuemu::launch(dim3((nBlocks + D1_WARPS(1) - 1) / D1_WARPS(1)), dim3(D1_WARPS(1) * 32), 0, [&] { zstd_dec_entropy_kernel<1>(src, srcSize, blocks.data(), nBlocks, lits.data(), hufTabs, litJobs, seqTabs, seqJobs); });
        cuemu::launch(dim3((nBlocks + 127u) / 128u), dim3(128), 0, [&] { zstd_dec_seq_streams_kernel(src, srcSize, blocks.data(), nBlocks, seqs.data(), seqTabs, seqJobs); });
    }
    const bool maybeJump = jumpMode == 2u || (jumpMode == 1u && (counts.maxFrameBlocks + B2Z_DEC_UNIT_BLOCKS - 1u) / B2Z_DEC_UNIT_BLOCKS >= B2Z_DEC_JUMP_MIN_UNITS);
    if (nFrames) cuemu::launch(dim3((nFrames + 127) / 128), dim3(128), 0, [&] { zstd_dec_frame_sizes_kernel(frames.data(), nFrames, blocks.data(), &counts, maybeJump ? jumpMode : 0u); });
    cuemu::launch(dim3(1), dim3(32), 0, [&] { zstd_dec_frame_offsets_kernel(frames.data(), nFrames, dstCap, &counts, &total); });
    if (nJumpOut) *nJumpOut = counts.nJump;
    if (getenv("B2Z_EMU_JUMP_DEBUG")) for (uint32_t f = 0; f < nFrames; f++) {
        uint32_t t[3] = {0, 0, 0}, firstNear = 0, firstComp = 0, anyNear = 0;
        for (uint32_t k = 0; k < frames[f].nBlocks; k++) { const DecBlock& b = blocks[frames[f].firstBlock + k]; t[b.type]++; anyNear += b.nearBehind;
            if (k && k % B2Z_DEC_UNIT_BLOCKS == 0) { firstComp += b.type == 2; firstNear += b.type == 2 && b.nearBehind; } }
        fprintf(stderr, "frame %u: blocks %u (raw %u rle %u comp %u) units %u firstComp %u firstNear %u anyNear %u jump %u\n", f, frames[f].nBlocks, t[0], t[1], t[2],
                (frames[f].nBlocks + B2Z_DEC_UNIT_BLOCKS - 1) / B2Z_DEC_UNIT_BLOCKS, firstComp, firstNear, anyNear, frames[f].jump);
    }
    if (maybeJump && !counts.status && counts.nJump && nBlocks && total) {             // launch_zstd_dec_jump
        const uint64_t seg = 1ull << g_emu_jump_seglog;
        std::vector<uint32_t> ptr((size_t)(total < seg ? total : seg) + 16, 0xCDCDCDCDu), flags(B2Z_DEC_JUMP_ROUNDS + 1u, 0u);
        std::vector<uint8_t> tileDone((size_t)(((total < seg ? total : seg) + 127) >> 7) + 1, 0);
        for (uint64_t S = 0; S < total; S += seg) {
            const uint64_t E = S + seg < total ? S + seg : total;
            std::fill(flags.begin(), flags.end(), 0u); std::fill(tileDone.begin(), tileDone.end(), (uint8_t)0);
            cuemu::launch(dim3((nBlocks + 3u) / 4u < 3u ? (nBlocks + 3u) / 4u : 3u), dim3(128), 0, [&] { zstd_dec_jump_build_kernel(src, frames.data(), blocks.data(), nBlocks, lits.data(), seqs.data(), dst, &counts, ptr.data(), S, E); });
            const uint64_t groups = (E - S + 3u) >> 2;
            const uint32_t grid = (uint32_t)((groups + 255u) / 256u < 2u ? (groups + 255u) / 256u : 2u);
            for (uint32_t r = 0; r < B2Z_DEC_JUMP_ROUNDS; r++)
                cuemu::launch(dim3(grid), dim3(256), 0, [&] { zstd_dec_jump_round_kernel<false>(frames.data(), nFrames, S, E, ptr.data(), flags.data(), tileDone.data(), r, dst, &counts); });
            cuemu::launch(dim3(grid), dim3(256), 0, [&] { zstd_dec_jump_round_kernel<true>(frames.data(), nFrames, S, E, ptr.data(), flags.data(), tileDone.data(), 0, dst, &counts); });
        }
    }
    if (nFrames) {
        std::vector<uint32_t> unitState((size_t)nBlocks / B2Z_DEC_UNIT_BLOCKS + nFrames + 2u, 0u);
        cuemu::launch(dim3(nFrames < 5u ? nFrames : 5u), dim3(32), 0, [&] { zstd_dec_exec_kernel(src, frames.data(), nFrames, blocks.data(), lits.data(), seqs.data(), dst, &counts, unitState.data()); });
        cuemu::launch(dim3((nFrames + 1) / 2), dim3(64), 0, [&] { zstd_dec_verify_kernel(src, frames.data(), nFrames, dst, &counts); });
    }
    return counts.status ? -(int64_t)counts.status : (int64_t)total;
}

// sha256_pieces_kernel: out[i] = 8 big-endian words per range
void emu_sha256_pieces(const uint8_t* src, const uint64_t* off, const uint64_t* len, uint32_t nPieces, uint32_t* out) {
    cuemu::launch(dim3((nPieces + 63u) / 64u), dim3(64), 0, [&] { sha256_pieces_kernel(src, off, len, nPieces, out); });
}

}
