/* b2z_params.h -- algorithm constants shared by the CUDA kernels and (read-only) by the
 * oracle restatement, so that both state the same algorithm.  Plain C, host+device. */
#ifndef B2Z_PARAMS_H
#define B2Z_PARAMS_H
#include <stdint.h>

#ifdef __CUDACC__
#define B2Z_HD __host__ __device__ __forceinline__
#else
#define B2Z_HD static inline
#endif

#define B2Z_DEF_FRAMELOG   20      /* independent zstd frame = 1 MiB of input                */
#define B2Z_DEF_HASHLOG_L  15      /* stage F: long (8-byte hash) table entries -- 128 KiB of the CTA's shared memory  */
#define B2Z_DEF_HASHLOG_S  14      /* stage F: short (5-byte hash) table entries -- 64 KiB of shared memory            */
#define B2Z_MAX_HASHLOG_SUM_WORDS 49152u  /* 2^L + 2^S entries must fit 192 KiB of shared memory                     */
#define B2Z_DEF_CHUNKLOG   7       /* stage F: positions whose table reads all precede their table writes (one "turn") */
#define B2Z_SEG            4096u   /* stage G: bytes parsed by one lane; matches never cross a segment end            */
#define B2Z_SEGLOG         12
/* stage G prices, in 1/16 bit: a match costs its offset's extra bits + B2Z_DP_MATCH + the extra bits of its length code;
 * a literal costs log2(total / count) of its byte in the block's sampled histogram, clamped */
#define B2Z_DP_MATCH       128u
#define B2Z_DP_NTRUNC      2u      /* a candidate of length L is also priced at L-1 .. L-NTRUNC                       */
#define B2Z_DP_MINLEN      4u
#define B2Z_DP_LIT_MIN     16u
#define B2Z_DP_LIT_MAX     192u
/* candidate word of one position (stage F / stage L -> stage G): 0 = none, else offset << 5 | length (length <= B2Z_CAP = 16,
 * offset < 2^27: the widest window of the long mode) */
#define B2Z_CAND(len, off) (((uint32_t)(off) << 5) | (uint32_t)(len))
#define B2Z_CAND_LEN(c)    ((c) & 31u)
#define B2Z_CAND_OFF(c)    ((c) >> 5)
/* bytes of a block that feed the literal histogram: the first 64 of every 256 */
#define B2Z_DP_SAMPLED(i)  ((((i) >> 6) & 3u) == 0u)
#define B2Z_MAX_FRAMELOG   24
/* long mode (B200Z_P_LONG, the reference's long=N / ZSTD_c_enableLongDistanceMatching, zstd_ldm.c): a frame of 8 windows (window <= 2^27) is
 * cut into REGIONS of 2^regionLog bytes, stage F's unit (its tables start empty in every region); stage L then looks, for one
 * position in 2^B2Z_LDM_RATELOG, for the first place of the frame that holds the same B2Z_LDM_MINMATCH bytes */
#define B2Z_DEF_PLAIN_REGIONLOG 19  /* outside the long mode: a 1 MiB frame is two regions.  Costs 0.2 % of ratio on text (2.3825 -> 2.3777: the
                                    * second region starts with empty tables) and halves the longest chain the decoder's execute stage has to
                                    * walk (its units are 4 blocks) */
#define B2Z_MAX_LONGLOG    27
#define B2Z_DEF_REGIONLOG  20
#define B2Z_LDM_MINMATCH   64u
#define B2Z_LDM_RATELOG    7u
#define B2Z_LDM_EPOCHLOG(windowLog) ((windowLog) - 1u)   /* stage L keeps one table per EPOCH of half a window: a position's own epoch and the two before it cover its window */
#define B2Z_LDM_LOG(windowLog) ((windowLog) - 6u)   /* entries of an epoch's sample table: four per sample of the epoch */
#define B2Z_LDM_TAGBITS    4u      /* entry = position in the epoch << 4 | tag, 0xFFFFFFFF = empty                       */
#define B2Z_LONG_FRAMELOG(windowLog) ((windowLog) + 3u > 30u ? 30u : (windowLog) + 3u)   /* long mode: a frame is 8 windows (at most 1 GiB) */
#define B2Z_CAP            16u     /* stage F compares at most this many bytes (two 8-byte words, no loop); stage G extends a chosen match of this length */
#define B2Z_MAXSEQ         32768u  /* raw sequences per 128 KiB block (min match 4)          */
#define B2Z_BLOCK          131072u
#define B2Z_FRAME_HDR_MAX  10
#define B2Z_LIT_HUF_MIN    64u     /* fewer literals than this are stored raw                */
#define B2Z_LIT_RLE_MIN    8u
#define B2Z_BODY_CAP       196608u /* a block body whose size upper bound exceeds this is stored raw */

/* final sequence record: offBase (28 bits) | litLength (18) | matchLength (18) */
#define B2Z_PACK_SEQ(offBase, ll, ml) ((uint64_t)(offBase) | ((uint64_t)(ll) << 28) | ((uint64_t)(ml) << 46))
#define B2Z_SEQ_OFFBASE(s) ((uint32_t)((s) & 0xFFFFFFFu))
#define B2Z_SEQ_LL(s)      ((uint32_t)(((s) >> 28) & 0x3FFFFu))
#define B2Z_SEQ_ML(s)      ((uint32_t)(((s) >> 46) & 0x3FFFFu))

/* ---- LZMA2 encoder (stage R: range coding of the stage-M sequences of one frame = one dictionary-reset block) ---- */
/* default literal / position context bits (B200Z_P_LZMA2_LC/LP/PB change them) */
#define B2Z_LZ2_LC 2u      /* 2 codes G2 text as well as 3 (2.3961 vs 2.3955) and halves the literal model: the whole model fits shared memory */
#define B2Z_LZ2_LP 0u
#define B2Z_LZ2_PB 2u
#define B2Z_LZ2_PROPS ((B2Z_LZ2_PB * 5u + B2Z_LZ2_LP) * 9u + B2Z_LZ2_LC)   /* 0x5D */
/* flags bit 15: the coders take lc / lp / pb from the properties byte (pb * 5 + lp) * 9 + lc in flags bits 16..23 (lc + lp <= 4,
 * pb <= 4) and run their run-time instantiations; clear: the defaults above, through the compile-time instantiations */
#define B2Z_FLAG_LZ2_PROPS 0x8000u
B2Z_HD uint32_t b2z_lz2_props(uint32_t flags) { return (flags & B2Z_FLAG_LZ2_PROPS) ? ((flags >> 16) & 0xFFu) : B2Z_LZ2_PROPS; }
B2Z_HD uint32_t b2z_lz2_lc(uint32_t props) { return props % 9u; }
B2Z_HD uint32_t b2z_lz2_lp(uint32_t props) { return (props / 9u) % 5u; }
B2Z_HD uint32_t b2z_lz2_pb(uint32_t props) { return props / 45u; }
/* literal model entries: 0x300 << (lc + lp) */
B2Z_HD uint32_t b2z_lz2_litn(uint32_t props) { return 0x300u << (b2z_lz2_lc(props) + b2z_lz2_lp(props)); }
#define B2Z_LZ2_PACK_LIMIT   (65536u - 64u)        /* a chunk is closed once this many packed bytes are pending (format max 64 KiB) */
#define B2Z_LZ2_UNPACK_LIMIT ((1u << 21) - 512u)   /* ... or this many input bytes are covered (format max 2 MiB)                 */
#define B2Z_LZ2_MAXLEN 273u
/* flags bits 8..10: log2 of the state-reset slices a frame's range coding is split into (0..3, clamped to the frame's blocks) */
#define B2Z_DEF_LZ2_SLICELOG 2u
#define B2Z_LZ2_SLICELOG(flags) (((flags) >> 8) & 7u)
#define B2Z_LZ2_SLICE_BLOCKS(frameLog, flags) \
    ((B2Z_LZ2_SLICELOG(flags) >= (frameLog) - 17u) ? 1u : (1u << ((frameLog) - 17u - B2Z_LZ2_SLICELOG(flags))))
/* worst-case bytes of one frame's chunk stream while it is being produced: every finished chunk is at most its input + 6
 * (raw fallback), a chunk covers >= 8 KiB of input (a literal costs < 7 bytes even with saturated models), plus the
 * chunk in flight */
#define B2Z_LZ2_FRAME_BOUND(n) ((n) + ((n) / 8192u + 2u) * 8u + 65536u + 128u)

/* flags bit 4: method 21 parses by price (stage C candidates + stage P dynamic programme) instead of the greedy stage M */
#define B2Z_FLAG_LZ2_OPT 0x10u
/* flags bit 5: the Zstandard encoder parses by price (stage C candidates + stage Z dynamic programme per block) instead of stage M */
#define B2Z_FLAG_ZSTD_OPT 0x20u
#define B2Z_ZSTD_OPT_LEVEL 8       /* B200Z_P_LEVEL at or above this selects it */
/* the level ladder below it (the strategies of clevels.h:27-50 as far as stage F has them):
 *   levels 1-2 and the fast levels: bit 6 -- only the short (5-byte hash) table, grown to 2^15 entries: the role of ZSTD_fast
 *   levels 3-4: both tables: ZSTD_dfast
 *   levels 5-7: bit 7 -- a position also sees the lower positions of its own 32-position step (two __match_any_sync per step):
 *               nearer candidates on data with short-distance repeats, for about twice stage F's time */
#define B2Z_FLAG_FIND_FAST 0x40u
#define B2Z_FLAG_FIND_STEP 0x80u
B2Z_HD uint32_t b2z_level_find_flags(int level) { return level <= 2 ? B2Z_FLAG_FIND_FAST : (level >= 5 && level < B2Z_ZSTD_OPT_LEVEL ? B2Z_FLAG_FIND_STEP : 0u); }

/* digests (b2z_crc.cu): reflected polynomials of CRC-32 (C/7zCrc.c) and CRC-64/XZ (C/XzCrc64.c) */
#define B2Z_CRC32_POLY 0xEDB88320u
#define B2Z_CRC64_POLY 0xC96C5795D7870F42ull

/* stage L: is position p (8 bytes v there) a sample, and the key of the 32 bytes there */
B2Z_HD int b2z_ldm_sampled(uint64_t v) { return ((v * 0x9E3779B185EBCA87ULL) >> (64 - B2Z_LDM_RATELOG)) == (1u << B2Z_LDM_RATELOG) - 1u; }   /* a run of zeros is never one */
B2Z_HD uint64_t b2z_ldm_key(uint64_t w0, uint64_t w1, uint64_t w2, uint64_t w3) {
    uint64_t k = w0 * 0xCF1BBCDCB7A56463ULL;
    k = (k ^ (k >> 29) ^ w1) * 0xCF1BBCDCB7A56463ULL; k = (k ^ (k >> 29) ^ w2) * 0xCF1BBCDCB7A56463ULL; k = (k ^ (k >> 29) ^ w3) * 0xCF1BBCDCB7A56463ULL;
    return k ^ (k >> 32);
}

/* multiplicative hashes: same constants as the reference (zstd_compress_internal.h:903-924) */
#define B2Z_PRIME5 889523592379ULL
#define B2Z_PRIME8 0xCF1BBCDCB7A56463ULL

#endif
