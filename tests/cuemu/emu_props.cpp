// emu_props.cpp -- TEST INFRASTRUCTURE ONLY: the run-time context-bit instantiations of the method-21 encoder kernels
// (lzma2_parse_kernel<true>, lzma2_enc_range_kernel<GLIT, 1, true>, lzma2_enc_range32_kernel<true>: lc / lp / pb from the
// properties byte in flags bits 16..23, B2Z_FLAG_LZ2_PROPS) compiled for the host through cuemu.h, as emu_kernels.cpp does for the
// default instantiations.  Built by tests/test_oracle_lzma2_props.py into a temporary directory; never part of libb200z.so.
#define B2Z_CUEMU 1
#include "cuemu.h"
#include "../../7-zip-zstd_b200/csrc/lzma2_parse.cu"
#include "../../7-zip-zstd_b200/csrc/lzma2_enc.cu"

using namespace b2z;

static EncGeom geom(uint32_t frameLog, uint32_t flags) {
    EncGeom g; memset(&g, 0, sizeof(g));
    g.frameLog = frameLog; g.windowLog = frameLog; g.hashLogL = B2Z_DEF_HASHLOG_L; g.hashLogS = B2Z_DEF_HASHLOG_S; g.chunkLog = B2Z_DEF_CHUNKLOG; g.flags = flags;
    return g;
}

extern "C" {

// stage C (lzma2_cand_kernel; independent of the context bits)
uint64_t emu_props_cand(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, uint32_t nWarps, uint32_t* cand) {
    const EncGeom g = geom(frameLog, flags);
    std::vector<uint32_t> tables((size_t)nWarps * lzma2_cand_table_words(frameLog), 0xCDCDCDCDu);
    return cuemu::launch(dim3(nWarps), dim3(32), 0, [&] { lzma2_cand_kernel(src, srcSize, g, tables.data(), cand); });
}

// stage P, run-time instantiation, shared memory sized for the setting as launch_lzma2_parse does; nseq zeroed here
uint64_t emu_props_parse(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, const uint32_t* cand, uint64_t* seqs, uint32_t* nseq) {
    if (!(flags & B2Z_FLAG_LZ2_PROPS)) return 0;
    const EncGeom g = geom(frameLog, flags);
    const uint64_t F = 1ull << frameLog;
    const uint32_t nFrames = (uint32_t)((srcSize + F - 1) >> frameLog), bpf = (uint32_t)(F >> 17);
    const uint32_t nChains = nFrames * (bpf / B2Z_LZ2_SLICE_BLOCKS(frameLog, flags));
    memset(nseq, 0, (size_t)nFrames * bpf * sizeof(uint32_t));
    return cuemu::launch(dim3(nChains), dim3(32), lzma2_parse_smem_bytes(flags), [&] { lzma2_parse_kernel<true>(src, srcSize, g, cand, seqs, nseq, nChains); });
}

// stage R, run-time instantiations (glit 0: model in shared memory, 1: literal model in global memory, 2: the lock-step kernel,
// lc + lp <= 3 only) + assembly -> the chunk stream with its end marker.  -1 slot overflow, -2 dst too small, -3 refused setting
int64_t emu_props_range_and_assemble(const uint8_t* src, uint64_t srcSize, uint32_t frameLog, uint32_t flags, const uint64_t* seqs, const uint32_t* nseq,
                                     uint8_t* dst, uint64_t dstCap, int glit) {
    const uint32_t props = b2z_lz2_props(flags);
    if (!(flags & B2Z_FLAG_LZ2_PROPS) || (glit == 2 && b2z_lz2_lc(props) + b2z_lz2_lp(props) > B2Z_R32_MAX_LCLP)) return -3;
    const EncGeom g = geom(frameLog, flags);
    const uint32_t nFrames = (uint32_t)((srcSize + (1ull << frameLog) - 1) >> frameLog);
    const uint32_t nChains = nFrames * lzma2_enc_slices_per_frame(g);
    const uint32_t stride = (uint32_t)lzma2_enc_slot_stride(g), LITN = b2z_lz2_litn(props);
    std::vector<uint8_t> slots((size_t)nChains * stride, 0xCD); std::vector<uint32_t> slotSize(nChains + 1, 0xCDCDCDCDu); uint32_t status = 0;
    std::vector<uint16_t> spill(glit == 1 ? (size_t)nChains * LITN : 1, 0xCDCD);
    std::vector<uint16_t> models(glit == 2 ? lzma2_enc_model_bytes(nChains, flags) / 2 : 1, 0xCDCD);
    if (glit == 2) cuemu::launch(dim3(((nChains + 31u) / 32u + B2Z_R32_WARPS - 1u) / B2Z_R32_WARPS), dim3(32 * B2Z_R32_WARPS), B2Z_R32_WARPS * B2Z_R32_QCAP * 32u * sizeof(uint16_t), [&] {
        lzma2_enc_range32_kernel<true>(src, srcSize, g, seqs, nseq, slots.data(), stride, slotSize.data(), models.data(), &status, nChains); });
    else if (glit) cuemu::launch(dim3((nChains + 1u) / 2u), dim3(64), 2u * P_LIT * sizeof(uint16_t), [&] {
        lzma2_enc_range_kernel<true, 1, true>(src, srcSize, g, seqs, nseq, slots.data(), stride, slotSize.data(), spill.data(), &status, nChains); });
    else cuemu::launch(dim3(nChains), dim3(32), ((size_t)P_LIT + LITN) * sizeof(uint16_t), [&] {
        lzma2_enc_range_kernel<false, 1, true>(src, srcSize, g, seqs, nseq, slots.data(), stride, slotSize.data(), nullptr, &status, nChains); });
    if (status) return -1;
    std::vector<uint64_t> off(nChains + 2); uint64_t outSize = 0;
    cuemu::launch(dim3(1), dim3(1024), 0, [&] { lzma2_enc_offsets_kernel(slotSize.data(), nChains, off.data(), &outSize); });
    if (outSize > dstCap) return -2;
    cuemu::launch(dim3(nChains, 4), dim3(256), 0, [&] { lzma2_enc_gather_kernel(slots.data(), stride, slotSize.data(), off.data(), nChains, dst); });
    return (int64_t)outSize;
}

}
