/* oracle.h -- C API of the CPU oracle (liboracle.so).  TEST INFRASTRUCTURE ONLY:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load it. */
#ifndef B2ZO_ORACLE_H
#define B2ZO_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

uint64_t b2zo_xxh64(const void *data, size_t len, uint64_t seed);
uint32_t b2zo_crc32(const void *data, size_t n);      /* crc_oracle.c: 7-Zip's CRC32 (C/7zCrc.c CrcCalc) */
uint64_t b2zo_crc64(const void *data, size_t n);      /* CRC-64/XZ (C/XzCrc64.c) */
/* filter_oracle.c: in-place delta / branch converters by 7-Zip method id; 0 ok, -1 unknown filter or bad property */
int b2zo_filter(uint32_t methodId, int enc, void *data, size_t n, uint32_t prop);

/* Decode every frame (zstd + skippable) in src; returns size or <0 (-1 corrupt, -2 dst too
 * small, -3 checksum, -4 dictionary needed). */
int64_t b2zo_zstd_decompress(void *dst, size_t dstCap, const void *src, size_t srcSize);

/* Encoder restatement: the exact algorithm the CUDA kernels implement (see zstd_enc_oracle.c).
 * Output is byte-identical to the GPU path for the same parameters. */
typedef struct {
    uint32_t frameLog;      /* log2 of independent frame size (default 22 = 4 MiB)            */
    uint32_t hashLogL;      /* stage F long (8-byte hash) table log (default 15)              */
    uint32_t hashLogS;      /* stage F short (5-byte hash) table log (default 14)             */
    uint32_t windowLog;     /* max match distance log (default = frameLog)                    */
    uint32_t chunkLog;      /* stage F: log2 positions per table turn (default 7)             */
    uint32_t flags;         /* bit0: skippable size hints before each frame; bit1: checksum;
                               bits 8..10: LZMA2 slice log; bit4: LZMA2 price-based parse */
    uint32_t regionLog;     /* long mode: stage F's unit inside a frame (0 = the frame)        */
    uint32_t ldmLog;        /* long mode: log2 entries of stage L's per-frame sample table (0 = no stage L) */
} b2zo_enc_params;

void   b2zo_enc_default_params(b2zo_enc_params *p, int level);
size_t b2zo_zstd_compress_bound(size_t srcSize, const b2zo_enc_params *p);
int64_t b2zo_zstd_compress(void *dst, size_t dstCap, const void *src, size_t srcSize, const b2zo_enc_params *p);

/* Stage tap for parity with the GPU's stage F: one candidate word per position of one frame (B2Z_CAND, b2z_params.h) */
void b2zo_zstd_candidates(const void *frame, uint32_t n, const b2zo_enc_params *p, uint32_t *cand);

/* Stage tap for parity with the GPU's stage G: per 128 KiB block, final sequences packed as
 * B2Z_PACK_SEQ(offBase, ll, ml) (b2z_params.h) and the literal bytes (at the block's offset). */
int64_t b2zo_zstd_find_sequences(const void *src, size_t srcSize, const b2zo_enc_params *p,
                                 uint64_t *seqs /* [nblocks*B2Z_MAXSEQ] */, uint32_t *nseq /* [nblocks] */,
                                 uint8_t *lits /* [srcSize] */, uint32_t *nlit /* [nblocks] */);

/* Stage tap for parity with the GPU's stage E: one block [blkStart, blkStart + blkSize) of `frame` coded from its sequences
 * (B2Z_PACK_SEQ) and literal bytes, with its 3-byte header (last = Last_Block flag).  Returns the bytes written (at most
 * blkSize + 3), -1 on a bad argument, -2 when dstCap < blkSize + 3. */
int64_t b2zo_zstd_encode_block(void *dst, size_t dstCap, const void *frame, size_t blkStart, size_t blkSize, int last,
                               const uint64_t *seqs, uint32_t nbSeq, const uint8_t *lits, uint32_t nlit);


/* ---- LZMA2 (method 21) decoder: lzma2_dec_oracle.c ---- */
/* raw LZMA2 chunk stream -> dst; dictProp = the coder's 1-byte property. returns size, -1 corrupt, -2 dst too small */
int64_t b2zo_lzma2_decompress(void *dst, size_t dstCap, const void *src, size_t srcSize, uint32_t dictProp, size_t *srcUsed);

/* ---- LZMA2 (method 21) encoder: lzma2_enc_oracle.c (sequential statement of the GPU encoder) ---- */
size_t  b2zo_lzma2_compress_bound(size_t srcSize, const b2zo_enc_params *p);
int64_t b2zo_lzma2_compress(void *dst, size_t dstCap, const void *src, size_t srcSize, const b2zo_enc_params *p, uint32_t *dictProp);

/* price-based parse (lzma2_opt_oracle.c; flags bit 4 of b2zo_lzma2_compress selects it).  Stage taps for parity with the GPU:
 * stage C: candidates of one frame, LZP_NCAND packed words per position (b2z_lzma_model.h);
 * stage P: one frame -> per-block sequences, block-indexed like b2zo_zstd_find_sequences (cand = stage C's output, or NULL) */
void b2zo_lzma2_candidates(const void *base, uint32_t n, uint32_t frameLog, uint32_t *cand);
void b2zo_lzma2_parse_frame(const void *base, uint32_t n, const b2zo_enc_params *P, const uint32_t *cand, uint64_t *seqs, uint32_t *nseq);

/* test taps: the coder model (probabilities [1848 + (0x300 << lc)], then state, rep0..3) at the end of a frame as stage R leaves it
 * after coding seqs (returns how often it initialised the model), and as stage P's simulation leaves it (last slice) */
int64_t b2zo_lzma2_final_model(const void *base, uint32_t n, const b2zo_enc_params *P, const uint64_t *seqs, const uint32_t *nseq, uint16_t *probsOut, uint32_t *ctxOut);
void b2zo_lzma2_parse_final_model(const void *base, uint32_t n, const b2zo_enc_params *P, uint64_t *seqs, uint32_t *nseq, uint16_t *probsOut, uint32_t *ctxOut);

/* price-based Zstandard parse (zstd_opt_oracle.c; flags bit 5 of b2zo_zstd_compress / b2zo_zstd_find_sequences selects it):
 * one frame -> per-block sequences and literal bytes, on stage C's candidates (cand, or NULL to compute them here) */
void b2zo_zstd_parse_frame(const void *base, uint32_t n, const b2zo_enc_params *P, const uint32_t *cand, uint64_t *seqs, uint32_t *nseq, uint8_t *lits, uint32_t *nlit);

#ifdef __cplusplus
}
#endif
#endif
