/* b2z_filter_ops.h -- the per-instruction rules of the stateless branch converters as arithmetic on one 32-bit word.
 * Plain C, host + device (B2Z_HD): used by csrc/b2z_filter.cu; the oracle (oracle/filter_oracle.c) states the same rules in its own
 * words and both are checked against the reference's converters (C/Bra.c via oracle/_ref/libref_xz.so) word by word.
 *
 * What the converters do (C/Bra.h:46-50): in CALL-type instructions the relative target becomes absolute (encode) or back
 * (decode), which makes repeated calls to one function byte-identical and so compressible.  `ia` = address of the instruction
 * (start offset property + position in the stream).  ARM64: C/Bra.c:75-123, ARM: :126-152, PPC: :155-191, SPARC: :198-252. */
#ifndef B2Z_FILTER_OPS_H
#define B2Z_FILTER_OPS_H
#include "b2z_params.h"

/* 7-Zip method ids of the filters (CPP/7zip/Compress/BranchRegister.cpp, DeltaFilter.cpp; DOC/Methods.txt) */
#define B200Z_F_DELTA 0x03u
#define B200Z_F_ARM64 0x0Au
#define B200Z_F_X86   0x03030103u
#define B200Z_F_PPC   0x03030205u
#define B200Z_F_ARM   0x03030501u
#define B200Z_F_ARMT  0x03030701u
#define B200Z_F_SPARC 0x03030805u
#define B200Z_F_RISCV 0x0Bu

B2Z_HD uint32_t b2z_bswap32(uint32_t v) { return (v >> 24) | ((v >> 8) & 0xFF00u) | ((v << 8) & 0xFF0000u) | (v << 24); }

/* w = the instruction as the CPU reads it (little endian for ARM / ARM64, big endian for PPC / SPARC) */
B2Z_HD uint32_t b2z_conv_arm64(uint32_t w, uint32_t ia, int enc) {
    if ((w >> 26) == 0x25u) {                                       /* BL imm26: word offset */
        const uint32_t t = ia >> 2, imm = enc ? w + t : w - t;
        return 0x94000000u | (imm & 0x03FFFFFFu);
    }
    if ((w & 0x9F000000u) == 0x90000000u) {                         /* ADRP: 21-bit page offset immhi:immlo */
        const uint32_t imm = ((w >> 3) & 0x1FFFFCu) | ((w >> 29) & 3u);
        const uint32_t biased = (imm + (1u << 17)) & 0x1FFFFFu;     /* only offsets in [-2^17, 2^17) pages are converted */
        if (biased < (1u << 18)) {
            const uint32_t page = ia >> 12;
            const uint32_t b2 = (enc ? biased + page : biased - page) & 0x3FFFFu;
            const uint32_t out = (b2 - (1u << 17)) & 0x1FFFFFu;     /* back to a sign-extended 21-bit offset */
            return (w & 0x9F00001Fu) | ((out & 3u) << 29) | ((out >> 2) << 5);
        }
    }
    return w;
}
B2Z_HD uint32_t b2z_conv_arm(uint32_t w, uint32_t ia, int enc) {
    if ((w >> 24) != 0xEBu) return w;                               /* BL imm24, relative to the instruction after next */
    const uint32_t t = (ia + 8u) >> 2, imm = enc ? w + t : w - t;
    return 0xEB000000u | (imm & 0x00FFFFFFu);
}
/* ARM Thumb BL (C/Bra.c:255-340): a pair of halfwords 11110 hhhhhhhhhhh, 11111 lllllllllll at a 2-byte aligned position; the 22-bit
 * halfword offset h:l is relative to the instruction address + 4.  Two such pairs cannot overlap (the second halfword of one would
 * have to start with both 11111 and 11110), so every position converts on its own.  h0 / h1: the halfwords, little endian. */
B2Z_HD int b2z_armt_is_bl(uint32_t h0, uint32_t h1) { return (h0 & 0xF800u) == 0xF000u && (h1 & 0xF800u) == 0xF800u; }
B2Z_HD void b2z_conv_armt(uint32_t *h0, uint32_t *h1, uint32_t ia, int enc) {
    const uint32_t off = ((*h0 & 0x7FFu) << 11) | (*h1 & 0x7FFu), t = (ia + 4u) >> 1;
    const uint32_t v = enc ? off + t : off - t;
    *h0 = 0xF000u | ((v >> 11) & 0x7FFu); *h1 = 0xF800u | (v & 0x7FFu);
}
B2Z_HD uint32_t b2z_conv_ppc(uint32_t w, uint32_t ia, int enc) {
    if ((w & 0xFC000003u) != 0x48000001u) return w;                 /* bl: AA = 0, LK = 1 */
    const uint32_t v = enc ? w + ia : w - ia;
    return 0x48000000u | (v & 0x03FFFFFFu);
}
B2Z_HD uint32_t b2z_conv_sparc(uint32_t w, uint32_t ia, int enc) {
    const uint32_t top = w >> 22;
    if (top != 0x100u && top != 0x1FFu) return w;                   /* call with a displacement in [-2^22, 2^22) words */
    const uint32_t biased = ((w & 0x3FFFFFu) + (top == 0x100u ? (1u << 22) : 0u)) << 2;      /* (disp + 2^22) * 4, < 2^25 */
    const uint32_t x = (enc ? biased + ia : biased - ia) & ((1u << 25) - 1u);
    return ((x - (1u << 24)) >> 2) | (1u << 30);
}

/* ---- x86 BCJ (C/Bra86.c:50-170).  CALL / JMP rel32 (E8 / E9) whose operand's top byte is 00 or FF become absolute.  A 3-bit history
 * of the opcode bytes just passed without a conversion (bit 2 = one byte back ... bit 0 = three back) vetoes or adjusts conversions.
 * The scan's state dies after three non-opcode bytes, so the buffer falls into CLUSTERS of opcode bytes (successive gaps <= 3) that
 * are converted independently of each other -- that is what the GPU parallelises over (b2z_filter.cu). */
B2Z_HD int b2z_x86_is_opcode(uint32_t b) { return (b & 0xFEu) == 0xE8u; }
B2Z_HD int b2z_x86_is_00_ff(uint32_t b) { b &= 0xFFu; return b == 0u || b == 0xFFu; }
/* one opcode byte at position i with history hist: returns 1 and the new operand if it is converted.  operand = the 4 bytes after
 * the opcode (little endian), next = address of the following instruction */
B2Z_HD int b2z_x86_convert(uint32_t hist, uint32_t operand, uint32_t next, int enc, uint32_t *out) {
    uint32_t fix = 0;
    if (hist == 0u) { if (!b2z_x86_is_00_ff(operand >> 24)) return 0; }
    else if (hist == 1u || hist == 2u || hist == 4u) {
        fix = hist >> 1;
        if (b2z_x86_is_00_ff(operand >> (8u * fix)) || !b2z_x86_is_00_ff(operand >> 24)) return 0;
    } else return 0;
    uint32_t v = operand + (1u << 24);
    v = enc ? v + next : v - next;
    if (hist != 0u && b2z_x86_is_00_ff(v >> (8u * fix))) { v ^= (0x100u << (8u * fix)) - 1u; v = enc ? v + next : v - next; }
    *out = (v & 0x1FFFFFFu) - (1u << 24);
    return 1;
}

/* ---- RISC-V (C/Bra.c:426-709).  A scan over even positions p with p + 8 <= (n & ~1) whose step (2, 4, 6 or 8 bytes) depends on the
 * instruction at p.  w0 / w1 = the little-endian words at p and p + 4, as they were BEFORE the scan wrote anything at or after p.
 *   JAL with rd = x1 / x5 (a call): its 21-bit offset becomes absolute, bits 20:1 stored big-endian over bytes 1.5 .. 3; step 4.
 *   AUIPC rd (rd not x0 / x2) followed by a 32-bit instruction whose rs1 = rd (auipc + jalr / load / addi): the pair's combined
 *     offset becomes absolute and is stored big-endian in the second word; the first becomes "AUIPC x2" holding the second
 *     instruction's low 20 bits; step 8.  Without such a partner: step 6 (the partner's slot is not looked at again as a start).
 *   AUIPC x0 / x2: a real "AUIPC x2" that looks like a converted pair (bits 13:12 = 3, bits 31:27 not x0 / x2) is escaped by
 *     swapping fields between its two words, so that decoding can tell the two apart; step 8.  Otherwise step 4.
 *   anything else: step 2.
 * The step is the same when encoding and when decoding (both read the same fields), and a conversion writes only inside
 * [p, p + step) -- so the positions the scan visits are a pure function of the input bytes.  b2z_filter.cu builds on that. */
/* -> the step at a position; bit 0 set = the position converts (JAL: w0 only; AUIPC: w0 and w1) */
B2Z_HD uint32_t b2z_riscv_scan(uint32_t w0, uint32_t w1) {
    const uint32_t op = w0 & 0x7Fu, rd = (w0 >> 7) & 0x1Fu;
    if (op == 0x6Fu) return (rd == 1u || rd == 5u) ? 5u : 2u;
    if (op != 0x17u) return 2u;
    if (rd != 0u && rd != 2u) return ((w1 & 3u) == 3u && ((w1 >> 15) & 0x1Fu) == rd) ? 9u : 6u;
    return (rd == 2u && ((w0 >> 12) & 3u) == 3u && ((w0 >> 27) & 0x1Du) != 0u) ? 9u : 4u;
}
B2Z_HD uint32_t b2z_riscv_jal_offset(uint32_t w) {                  /* the J-immediate, bits 20:1 (unsigned) */
    return ((w >> 11) & 0x100000u) | ((w >> 20) & 0x7FEu) | ((w >> 9) & 0x800u) | (w & 0xFF000u);
}
/* a converting position (b2z_riscv_scan bit 0) at address ia: rewrites *w0 (and *w1 for the 8-byte forms) */
B2Z_HD void b2z_riscv_enc(uint32_t *w0, uint32_t *w1, uint32_t ia) {
    const uint32_t a = *w0, b = *w1;
    if ((a & 0x7Fu) == 0x6Fu) {
        const uint32_t t = b2z_riscv_jal_offset(a) + ia;
        *w0 = (a & 0xFFFu) | (((t >> 17) & 0xFu) << 12) | (((t >> 9) & 0xFFu) << 16) | (((t >> 1) & 0xFFu) << 24);
    } else if (((a >> 7) & 0x1Fu) != 2u) {                          /* auipc rd + partner -> "auipc x2 | partner" + absolute target */
        *w0 = (b << 12) | (2u << 7) | 0x17u;
        *w1 = b2z_bswap32((a & 0xFFFFF000u) + (uint32_t)((int32_t)b >> 20) + ia);
    } else {                                                        /* escape a real auipc x2 */
        *w0 = ((a >> 27) << 7) | 0x17u | (b & 0xFFFFF000u);
        *w1 = (a >> 12) | (b << 20);
    }
}
B2Z_HD void b2z_riscv_dec(uint32_t *w0, uint32_t *w1, uint32_t ia) {
    const uint32_t a = *w0, b = *w1;
    if ((a & 0x7Fu) == 0x6Fu) {
        const uint32_t off = ((((a >> 12) & 0xFu) << 17) | (((a >> 16) & 0xFFu) << 9) | (((a >> 24) & 0xFFu) << 1)) - ia;
        *w0 = (a & 0xFFFu) | ((off & 0x100000u) << 11) | ((off & 0x7FEu) << 20) | ((off & 0x800u) << 9) | (off & 0xFF000u);
    } else if (((a >> 7) & 0x1Fu) == 2u) {                          /* a converted pair: rebuild auipc rd + partner */
        const uint32_t t = b2z_bswap32(b) - ia;
        *w0 = ((a >> 27) << 7) | 0x17u | ((t + 0x800u) & 0xFFFFF000u);
        *w1 = (a >> 12) | (t << 20);
    } else {                                                        /* an escaped auipc x2 */
        *w0 = (b << 12) | (2u << 7) | 0x17u;
        *w1 = (a & 0xFFFFF000u) | (b >> 20);
    }
}

#endif
