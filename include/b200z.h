/* b200z.h -- C ABI of libb200z.so: the H100 block-parallel codec engine behind 7-Zip's
 * ZSTD (method 4F71101) and LZMA2/FLZMA2 (method 21) coders.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types.  The host-side
 * coder classes (7-zip-zstd_b200/codec/, mirroring CPP/7zip/Compress/ZstdEncoder.cpp etc.) and
 * any other FFI (ctypes, cgo, JNI) bind exactly these entry points.
 *
 * Which reference interface each entry point replaces (paths under /root/reference):
 *   b200z_create / b200z_destroy ........ ZSTD_createCCtx / ZSTD_freeCCtx as used by
 *                                         CPP/7zip/Compress/ZstdEncoder.cpp:262-265, ZstdDecoder.cpp:76-80
 *   b200z_set_param ..................... ZSTD_CCtx_setParameter calls, ZstdEncoder.cpp:268-396
 *   b200z_zstd_compress_bound ........... ZSTD_compressBound (C/zstd/zstd.h)
 *   b200z_zstd_compress_{host,device} ... the ZSTD_compressStream2 loop of ZstdEncoder.cpp:398-461
 *                                         (one call = one whole Code() input; the zstdmt job slicing of
 *                                         C/zstd/zstdmt_compress.c:1184-1246 is the frame slicing here)
 *   b200z_zstd_decompress_{host,device} . the ZSTD_decompressStream loop of ZstdDecoder.cpp:108-173
 *   b200z_zstd_frame_info ............... ZSTD_getFrameHeader / ZSTD_findFrameCompressedSize
 *   b200z_last_error .................... ZSTD_getErrorName (ZstdEncoder.cpp:427-441 maps codes to HRESULT)
 *
 * All functions return B200Z_OK (0) or a negative B200Z_E_* code.  There is NO CPU fallback:
 * without a usable CUDA device every call fails with B200Z_E_NODEVICE.
 */
#ifndef B200Z_H
#define B200Z_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200Z_OK            0
#define B200Z_E_NODEVICE   -1   /* no CUDA device / driver error                          */
#define B200Z_E_MEMORY     -2   /* device or pinned-host allocation failed  (E_OUTOFMEMORY) */
#define B200Z_E_PARAM      -3   /* bad parameter                             (E_INVALIDARG)  */
#define B200Z_E_DSTSIZE    -4   /* destination too small                                     */
#define B200Z_E_CORRUPT    -5   /* malformed compressed data                 (S_FALSE)       */
#define B200Z_E_UNSUPPORTED -6  /* valid but unsupported input (dictionary, legacy frame) (E_NOTIMPL) */
#define B200Z_E_CUDA       -7   /* kernel launch / execution error           (E_FAIL)        */
#define B200Z_E_CHECKSUM   -8   /* content checksum mismatch                 (S_FALSE)       */

/* parameters (b200z_set_param) */
#define B200Z_P_LEVEL       1   /* 1..22.  Stage F + stage G with the finder's rung chosen as ZSTD_getCParams picks a strategy (clevels.h:27-50): 1-2 the short table
                                   alone (ZSTD_fast's role), 3-4 both tables (ZSTD_dfast), 5-7 both + the lower lanes of a position's own step (nearer candidates, twice
                                   the finder time); 8-22: the price-based parse on stage C's candidates (sets B200Z_P_ZSTD_PARSE) */
#define B200Z_P_FRAMELOG    2   /* log2 of the independent frame ("job") size, 17..24, default 20       */
#define B200Z_P_HASHLOG_L   3   /* stage F: log2 entries of the long (8-byte hash) table, 8..15, default 15; both tables live in one SM's shared memory */
#define B200Z_P_HASHLOG_S   4   /* stage F: log2 entries of the short (5-byte hash) table, 8..15, default 14 (2^L + 2^S <= 49152)       */
#define B200Z_P_WINDOWLOG   5   /* max match distance log, default = frameLog                            */
#define B200Z_P_FLAGS       6   /* bit0: skippable size hint before each frame (mcmilk MT convention; default on)
                                   bit1: XXH64 content checksum per frame (ZstdHandler.cpp:275 sets it for .zst) */
#define B200Z_P_BATCH_LOG   7   /* log2 of bytes compressed per kernel batch, default 31 (2 GiB; scratch = 9.5 x that) */
#define B200Z_P_CHUNKLOG    9   /* stage F: log2 positions per table turn (reads of a chunk precede its writes), 5..8, default 7 */
#define B200Z_P_LZMA2_MODEL 10  /* LZMA2 coders, where the probability models live: literal model in 1 = shared memory (13 warps/SM), 2 = global memory (32 warps/SM),
                                   0 = by block / chain count (default).  Encoder only: 3 = 32 chains per warp coded in lock-step from per-lane decision queues,
                                   models in global memory (same bytes; experimental -- slower than one chain per warp so far, csrc/lzma2_enc.cu) */
#define B200Z_P_LZMA2_SLICELOG 11 /* LZMA2 encoder: log2 of the state-reset slices a block's range coding is split into (0..3, default 2):
                                   independent range-coder chains per block, as fast-lzma2's encoder threads (lzma2_enc.c:1937) */
#define B200Z_P_LZMA2_PARSE 12  /* LZMA2 encoder parse: 0 = greedy/lazy on the finder shared with the zstd path (default), 1 = price-based:
                                   nearest-occurrence candidates by 3/4/6/8-byte keys + a windowed dynamic programme over the adaptive
                                   model -- the role of LzmaEnc.c:1225 GetOptimum / fast-lzma2 lzma2_enc.c:949 LZMA_optimalParse */
#define B200Z_P_ZSTD_PARSE  13  /* Zstandard encoder parse: 0 = stage F + stage G (shared-memory dual-hash finder, minimum-price path per 4 KiB segment), 1 = price-based: nearest-occurrence
                                   candidates + a per-block dynamic programme over adaptive code statistics -- the role of
                                   zstd_opt.c:1077 ZSTD_compressBlock_opt_generic.  B200Z_P_LEVEL sets it (>= 8); set it after the level to override */
#define B200Z_P_LONG        14  /* Zstandard encoder, long mode (the reference's long=N: ZstdEncoder.cpp:128-146 -> ZSTD_c_enableLongDistanceMatching + windowLog N,
                                   zstd_ldm.c): 0 = off (default), 21..27 = window of 2^N bytes in frames of 8 windows (at most 1 GiB).  A frame is cut into
                                   1 MiB regions, stage F's unit; stage L finds matches of >= 64 bytes up to a window back through tables of content-chosen
                                   samples.  The parse is stage G's at every level (the price-based stage C + Z works on frames of <= 16 MiB).
                                   Sets FRAMELOG and WINDOWLOG; set B200Z_P_FRAMELOG afterwards to leave the mode */
#define B200Z_P_REGIONLOG   15  /* Zstandard encoder: log2 of the finder's unit inside a frame (stage F starts with empty tables in every region, so no match
                                   crosses a region start: regions decode as independent chains), 17..FRAMELOG; 0 = the frame */
#define B200Z_P_DEC_JUMP    16  /* Zstandard decoder: which frames are resolved by pointer jumping (stage J: one pointer per output byte, doubled until it names a
                                   literal) instead of by execution units: 0 = none, 1 = frames of >= 8 units (4 MiB) whose units copy from one another -- the single
                                   sliding-window frame the reference's encoder writes (default), 2 = every frame (tests) */
#define B200Z_P_DEC_JUMP_SEGLOG 17 /* stage J resolves the output in segments of 2^this bytes, in order (16..30, default 30: 4 GiB of pointers at most, frames of any size) */
#define B200Z_P_HOST_BATCH_LOG 8 /* log2 of bytes per H2D|kernels|D2H pipeline batch of the *_host calls, default 30 (the decoder takes twice that) */
#define B200Z_P_LZMA2_LC    18  /* LZMA2 encoder: literal context bits lc, 0..4 (default 2)                                                       */
#define B200Z_P_LZMA2_LP    19  /* LZMA2 encoder: literal position bits lp, 0..4 (default 0); lc + lp <= 4 is checked when a compression starts   */
#define B200Z_P_LZMA2_PB    20  /* LZMA2 encoder: position bits pb, 0..4 (default 2).  lc/lp/pb travel in the chunk headers' properties byte
                                   (pb * 5 + lp) * 9 + lc; values other than 2/0/2 run the run-time instantiations of stages P and R.
                                   LZMA2_MODEL 3 codes lc + lp <= 3 only.  The reference's encoders default to lc3 (lc2 codes text as well here) */

/* statistics (b200z_get_stat): device milliseconds accumulated since the last b200z_reset_stats,
 * measured with CUDA events on the context's stream around each stage */
#define B200Z_S_ENC_MATCH_MS    1   /* the finder: stage F (or stage C of the price-based parses) */
#define B200Z_S_ENC_ENTROPY_MS  2
#define B200Z_S_ENC_ASSEMBLE_MS 3
#define B200Z_S_DEC_ENTROPY_MS  4
#define B200Z_S_DEC_EXEC_MS     5
#define B200Z_S_KERNEL_LAUNCHES 6   /* number of kernels launched */
#define B200Z_S_H2D_BYTES       7
#define B200Z_S_D2H_BYTES       8
#define B200Z_S_DEC_PREPASS_MS  9
#define B200Z_S_ENC_PARSE_MS    10  /* the parse: stage G (or stage P / stage Z of the price-based parses) */
#define B200Z_S_DEC_JUMP_FRAMES 11  /* Zstandard frames the decoder resolved by pointer jumping (stage J) */

typedef struct b200z_ctx b200z_ctx;

int  b200z_device_count(void);
int  b200z_create(b200z_ctx **out, int device);
/* One context over several devices of the box (devices[0] is the primary).  b200z_zstd_compress_host / b200z_zstd_decompress_host --
 * what ICompressCoder::Code() calls -- then deal batches of whole frames round-robin to the devices, each with its own streams,
 * staging and scratch, and write the output in input order: the bytes do not depend on the device count.  The other entry points
 * (device pointers, method 21, digests) run on the primary.  Replaces the worker pool of ZSTDMT_createCompressionJob /
 * ZSTDMT_flushProduced (C/zstd/zstdmt_compress.c:1403,1488) and MtCoder_Code (C/MtCoder.c:445) one level up. */
int  b200z_create_multi(b200z_ctx **out, const int *devices, int nDevices);
int  b200z_device_list(b200z_ctx *ctx, int *devices, int cap);          /* returns the number of devices of the context */
void b200z_destroy(b200z_ctx *ctx);
int  b200z_set_param(b200z_ctx *ctx, int param, int64_t value);
int  b200z_get_param(b200z_ctx *ctx, int param, int64_t *value);
const char *b200z_last_error(b200z_ctx *ctx);
double b200z_get_stat(b200z_ctx *ctx, int stat);
void b200z_reset_stats(b200z_ctx *ctx);

size_t b200z_zstd_compress_bound(b200z_ctx *ctx, size_t srcSize);

/* src/dst are DEVICE pointers (src 16-byte aligned); synchronous on the context's stream */
int b200z_zstd_compress_device(b200z_ctx *ctx, const void *d_src, size_t srcSize,
                               void *d_dst, size_t dstCap, size_t *dstSize);
/* src/dst are HOST pointers (pinned or pageable): H2D copy, compress, D2H copy */
int b200z_zstd_compress_host(b200z_ctx *ctx, const void *src, size_t srcSize,
                             void *dst, size_t dstCap, size_t *dstSize);

/* Many independent files in one call (the per-file fan-out of a non-solid archive: 7zEncode.cpp:325-332 runs one Code() per
 * file).  src: the files back to back, sizes[i] bytes each.  File i becomes its own run of 128 KiB frames at
 * dst[dstOffsets[i] .. dstOffsets[i+1]) -- byte-identical to compressing it alone with FRAMELOG 17 -- and decodes alone;
 * b200z_zstd_decompress_host on the whole output returns the files back to back.  An empty file yields zero bytes. */
size_t b200z_zstd_compress_batch_bound(b200z_ctx *ctx, size_t totalBytes, uint32_t nFiles);
int b200z_zstd_compress_batch_host(b200z_ctx *ctx, const void *src, const uint64_t *sizes, uint32_t nFiles,
                                   void *dst, size_t dstCap, uint64_t *dstOffsets /* [nFiles + 1] */);

/* Sum of the decompressed sizes of all frames in a host buffer (needs frame content sizes or
 * cheap block-header walks; returns B200Z_E_UNSUPPORTED if a frame's size is not declared). */
int b200z_zstd_frame_info(const void *src, size_t srcSize, uint64_t *contentSize, uint32_t *nFrames);

/* For callers that read a packed stream piece by piece (the coder module's decoder): the complete frames at the start of a buffer
 * that may end inside a frame.  *usedBytes = end of the last complete frame taken, *contentBound = the bytes they decode to (exact
 * where declared, else an upper bound from the block headers: raw / RLE size fields, 128 KiB per compressed block); stops before a
 * frame that would take the sum past maxContent unless it is the first.  B200Z_E_CORRUPT if the bytes at a frame start are no frame
 * or a frame's headers are malformed.  All three outputs are written on every return: on B200Z_E_CORRUPT they describe the complete
 * frames in front of the damage. */
int b200z_zstd_frame_prefix(const void *src, size_t srcSize, uint64_t maxContent, size_t *usedBytes, uint64_t *contentBound, uint32_t *nFrames);

int b200z_zstd_decompress_device(b200z_ctx *ctx, const void *d_src, size_t srcSize,
                                 void *d_dst, size_t dstCap, size_t *dstSize);
int b200z_zstd_decompress_host(b200z_ctx *ctx, const void *src, size_t srcSize,
                               void *dst, size_t dstCap, size_t *dstSize);

/* Test taps: run only the finder + parse (stage F + stage G, or stage C + stage Z) on a device buffer and copy the per-block
 * outputs to host arrays (same layout as the oracle's b2zo_zstd_find_sequences); stage_f: stage F's candidate words, one per
 * input byte (layout of b2zo_zstd_candidates, frames back to back). */
int b200z_zstd_enc_stage_m(b200z_ctx *ctx, const void *d_src, size_t srcSize,
                           uint64_t *seqs, uint32_t *nseq, uint8_t *lits, uint32_t *nlit);
int b200z_zstd_enc_stage_f(b200z_ctx *ctx, const void *d_src, size_t srcSize, uint32_t *cand);
/* stage_e: stage E (the entropy coder) alone, on the device buffer d_src and per-block sequences and literals from host arrays in
 * the layout of b2zo_zstd_find_sequences (seqs[b * 32768 + i] packed by B2Z_PACK_SEQ, block b's literals at lits + b * 128 KiB);
 * the finished blocks (3-byte header included) are written to dst back to back, their sizes to slotSize[b].  dstCap must cover
 * every block's raw size + 3. */
int b200z_zstd_enc_stage_e(b200z_ctx *ctx, const void *d_src, size_t srcSize, const uint64_t *seqs, const uint32_t *nseq,
                           const uint8_t *lits, const uint32_t *nlit, void *dst, size_t dstCap, uint32_t *slotSize);

/* ---- non-solid .7z archives of many files in one pass (BASELINE configs[4]; csrc/sevenz_api.cu) ----------------------------------
 * The reference's archive layer runs one Code() per file, strictly one after the other (CPP/7zip/Archive/7z/7zUpdate.cpp:2739-2810,
 * 7zEncode.cpp:482-487).  b200z_zstd_compress_batch_crc_host is b200z_zstd_compress_batch_host that also returns every file's CRC32
 * (CrcCalc) from the same bytes in HBM; b200z_7z_write_archive_host compresses all files in one GPU pass and writes the container
 * around them -- signature header, packed streams, uncompressed header: one folder per non-empty file, coder 04F71101 with its 5
 * property bytes, unpack sizes, CRCs, names (UTF-8 in, UTF-16LE in the archive), optional mtimes (Windows FILETIME) -- the layout of
 * 7zOut.cpp (WriteHeader :520-820) / DOC/7zFormat.txt.  b200z_7z_build_archive is the container writer alone (host code, no GPU):
 * packed = the packed streams of the non-empty files back to back. */
int b200z_zstd_compress_batch_crc_host(b200z_ctx *ctx, const void *src, const uint64_t *sizes, uint32_t nFiles,
                                       void *dst, size_t dstCap, uint64_t *dstOffsets, uint32_t *crcs);
size_t b200z_7z_archive_bound(b200z_ctx *ctx, size_t totalBytes, uint32_t nFiles, size_t namesBytes);
int b200z_7z_build_archive(const void *packed, const uint64_t *packSizes, const uint64_t *unpackSizes, const uint32_t *crcs, const char *const *names,
                           const uint64_t *mtimes, uint32_t nFiles, uint32_t level, void *dst, size_t dstCap, size_t *dstSize);
int b200z_7z_write_archive_host(b200z_ctx *ctx, const void *src, const uint64_t *sizes, const char *const *names, const uint64_t *mtimes, uint32_t nFiles,
                                void *dst, size_t dstCap, size_t *dstSize);

/* ---- LZMA2 / FLZMA2 (method 21) decoder --------------------------------------------------------------
 * src is the raw LZMA2 chunk stream a 7z folder stores for coder 21 (chunks ... 0x00 end marker); dictProp is the
 * coder's 1-byte property (0..40).  Replaces NCompress::NLzma2::CDecoder::Code -> Lzma2DecMt_Decode
 * (CPP/7zip/Compress/Lzma2Decoder.cpp:95-200, C/Lzma2DecMt.c:802) and Lzma2Decode (C/Lzma2Dec.c:452).
 * Parallel unit: every run of chunks that starts with a dictionary reset (control 0x01 / >= 0xE0), as in
 * Lzma2DecMt_MtCallback_Parse (C/Lzma2DecMt.c:237).  A stream with a single reset decodes on a single warp. */
int b200z_lzma2_stream_info(const void *src, size_t srcSize, uint64_t *contentSize, uint32_t *nBlocks, size_t *srcUsed);
/* For callers that read the packed stream piece by piece: the complete dictionary-reset blocks at the start of a buffer that may end
 * inside a chunk.  *usedBytes = the boundary (past the end marker when *ended), *contentSize = what the blocks before it decode to;
 * stops at the first boundary at or beyond maxContent.  The caller decodes [0, usedBytes) with a 0x00 end marker appended when !*ended. */
int b200z_lzma2_stream_prefix(const void *src, size_t srcSize, uint64_t maxContent, size_t *usedBytes, uint64_t *contentSize, uint32_t *nBlocks, int *ended);
int b200z_lzma2_decompress_device(b200z_ctx *ctx, const void *d_src, size_t srcSize, uint32_t dictProp,
                                  void *d_dst, size_t dstCap, size_t *dstSize);
int b200z_lzma2_decompress_host(b200z_ctx *ctx, const void *src, size_t srcSize, uint32_t dictProp,
                                void *dst, size_t dstCap, size_t *dstSize);

/* ---- LZMA2 / FLZMA2 (method 21) encoder --------------------------------------------------------------
 * Writes a raw LZMA2 chunk stream (+ end marker) of independent dictionary-reset blocks, one per 2^FRAMELOG input bytes,
 * and returns the 1-byte coder property for the 7z folder (what ICompressWriteCoderProperties emits,
 * Lzma2Encoder.cpp:117-121 / FastLzma2 :353-364).  Replaces NCompress::NLzma2::CEncoder::Code -> Lzma2Enc_Encode2
 * (Lzma2Encoder.cpp:124-134, C/Lzma2Enc.c:717) and CFastEncoder::Code -> FL2_compressStream (Lzma2Encoder.cpp:280-340,
 * C/fast-lzma2/fl2_compress.c).  lc/lp/pb are B200Z_P_LZMA2_LC/LP/PB (default 2/0/2); B200Z_E_PARAM when lc + lp > 4, or with
 * B200Z_P_LZMA2_MODEL 3 when lc + lp > 3 (Lzma2Enc_SetProps, Lzma2Enc.c:471). */
size_t b200z_lzma2_compress_bound(b200z_ctx *ctx, size_t srcSize);
int b200z_lzma2_compress_device(b200z_ctx *ctx, const void *d_src, size_t srcSize, void *d_dst, size_t dstCap,
                                size_t *dstSize, uint32_t *dictProp);
int b200z_lzma2_compress_host(b200z_ctx *ctx, const void *src, size_t srcSize, void *dst, size_t dstCap,
                              size_t *dstSize, uint32_t *dictProp);

/* Test tap of the price-based parse (B200Z_P_LZMA2_PARSE = 1): stage C's candidate words (4 per input byte) and stage P's
 * per-block sequences of a device buffer, layouts of the oracle's b2zo_lzma2_candidates / b2zo_lzma2_parse_frame. */
int b200z_lzma2_enc_stage_cp(b200z_ctx *ctx, const void *d_src, size_t srcSize, uint32_t *cand, uint64_t *seqs, uint32_t *nseq);

/* ---- digests of the archive layer on the GPU (SURVEY.md 8(f) item 4) -------------------------------------------------------
 * CRC32 as C/7zCrc.c:298 CrcCalc returns it (file / folder digests, CPP/7zip/Common/InStreamWithCRC.cpp) and CRC-64/XZ as
 * C/XzCrc64.c computes it (xz block check).  *_combine: crc(A || B) from crc(A), crc(B), |B| -- host arithmetic, no device. */
int b200z_crc32_device(b200z_ctx *ctx, const void *d_src, size_t n, uint32_t *crc);
int b200z_crc64_device(b200z_ctx *ctx, const void *d_src, size_t n, uint64_t *crc);
int b200z_crc32_host(b200z_ctx *ctx, const void *src, size_t n, uint32_t *crc);
int b200z_crc64_host(b200z_ctx *ctx, const void *src, size_t n, uint64_t *crc);
uint32_t b200z_crc32_combine(uint32_t crcA, uint32_t crcB, uint64_t lenB);
uint64_t b200z_crc64_combine(uint64_t crcA, uint64_t crcB, uint64_t lenB);

/* ---- .xz container around the LZMA2 coder (SURVEY.md 8(f) item 2) ----------------------------------------------------------
 * Replaces NCompress::NXz::CEncoder / CDecoder (CPP/7zip/Compress/XzEncoder.cpp, XzDecoder.cpp) -> Xz_Encode (C/XzEnc.c:1236) /
 * XzDecMt_Decode (C/XzDec.c).  The reader takes Blocks whose filter chain is LZMA2, optionally behind Delta / x86 / PowerPC / ARM / ARM Thumb / SPARC /
 * ARM64 / RISC-V filters (undone on the GPU; IA64 is B200Z_E_UNSUPPORTED); the writer emits LZMA2, optionally behind one of those filters (applied on the GPU per Block).  The writer emits one Block per 2^FRAMELOG input
 * bytes with both sizes in the Block header (the layout multi-threaded xz coders write); check type 0 none, 1 CRC32, 4 CRC64
 * (XZ_CHECK_*, C/Xz.h:31-35).  b200z_xz_wrap / b200z_xz_parse are the host-side container logic alone (no device needed). */
typedef struct {
    uint64_t packOff, packSize;      /* the Block's LZMA2 chunk stream inside the file, end marker included */
    uint64_t unpackSize, check;      /* decoded size; stored check value (low bytes first; 0 when none / longer than 8 bytes) */
    uint32_t dictProp, checkType;
    uint32_t nFilters;               /* filters in front of LZMA2 (0..3), in encoding order, as 7-Zip method ids for b200z_filter_* */
    uint32_t filterId[3], filterProp[3];
} b200z_xz_block;
size_t b200z_xz_wrap_bound(size_t lzma2Size, uint32_t nBlocks);
int b200z_xz_wrap(const void *lzma2, size_t lzma2Size, uint32_t dictProp, uint32_t checkType, const uint64_t *checks, uint32_t nChecks,
                  uint32_t filterId, uint32_t filterProp, void *dst, size_t dstCap, size_t *dstSize);
int b200z_xz_parse(const void *src, size_t srcSize, b200z_xz_block *blocks, uint32_t cap, uint32_t *nBlocks, uint64_t *contentSize);
size_t b200z_xz_compress_bound(b200z_ctx *ctx, size_t srcSize);
int b200z_xz_compress_host(b200z_ctx *ctx, const void *src, size_t srcSize, void *dst, size_t dstCap, size_t *dstSize, uint32_t checkType,
                           uint32_t filterId /* 0, or a b200z_filter_* id applied per Block in front of LZMA2 */, uint32_t filterProp);
int b200z_xz_decompress_host(b200z_ctx *ctx, const void *src, size_t srcSize, void *dst, size_t dstCap, size_t *dstSize);

/* ---- pre/post filters of a 7z folder / xz filter chain on the GPU (SURVEY.md 8(f) item 3) -----------------------------------
 * In place.  methodId = 7-Zip's filter id: 0x03 Delta (prop = distance 1..256; CPP/7zip/Compress/DeltaFilter.cpp, C/Delta.c),
 * 0x03030103 x86 BCJ (C/Bra86.c), 0x0A ARM64, 0x03030501 ARM, 0x03030701 ARM Thumb, 0x03030205 PPC, 0x03030805 SPARC, 0x0B RISCV (prop = start offset,
 * even for RISCV and ARM Thumb; BranchMisc.cpp -> C/Bra.c z7_BranchConv_*; an odd RISCV offset is B200Z_E_UNSUPPORTED; no alignment
 * requirement on the RISCV buffer).  BCJ2 and IA64 return B200Z_E_UNSUPPORTED. */
int b200z_filter_device(b200z_ctx *ctx, uint32_t methodId, int encode, void *d_data, size_t n, uint32_t prop);
int b200z_filter_host(b200z_ctx *ctx, uint32_t methodId, int encode, void *data, size_t n, uint32_t prop);

/* device memory helpers so FFI users need no CUDA binding of their own */
int b200z_dev_alloc(b200z_ctx *ctx, void **d_ptr, size_t bytes);
int b200z_dev_free(b200z_ctx *ctx, void *d_ptr);
int b200z_dev_upload(b200z_ctx *ctx, void *d_dst, const void *src, size_t bytes);
int b200z_dev_download(b200z_ctx *ctx, void *dst, const void *d_src, size_t bytes);
int b200z_host_alloc_pinned(void **ptr, size_t bytes);
int b200z_host_free_pinned(void *ptr);

#ifdef __cplusplus
}
#endif
#endif
