/* riscv_oracle.c -- TEST INFRASTRUCTURE ONLY: a sequential statement of the RISC-V branch converter that csrc/b2z_filter.cu runs on the
 * GPU (riscv_*_kernel).  Written from the filter's definition in plain loops; tests/test_riscv_filter.py compiles it into a temporary
 * library and checks it against the reference's own converter (C/Bra.c z7_BranchConv_RISCV_Enc / _Dec in oracle/_ref/libref_xz.so).
 *
 * RISC-V (7-Zip method 0x0B, xz filter 0x0B; C/Bra.h:73 -- little endian, 2-byte alignment, 6 bytes of look-ahead).  One pass over the
 * even offsets i with i + 8 <= (n rounded down to even); what happens at i depends on the instruction there (opcode = low 7 bits,
 * rd = bits 11:7), and the next offset is i + 2, 4, 6 or 8:
 *   JAL whose rd is a link register (ra = x1, t0 = x5): the target (address + J-offset) replaces the offset -- bits 20:17 of the
 *     target in the high nibble of byte 1, bits 16:9 in byte 2, bits 8:1 in byte 3; the opcode, rd and bits 11:8 stay.  Next: i + 4.
 *     Decoding reads the target back and stores address-relative J-offset fields again.
 *   AUIPC rd, rd neither x0 nor x2, followed by a 32-bit instruction (low bits 11) that reads rd as rs1 (bits 19:15): the pair is one
 *     PC-relative reference, upper 20 bits + the partner's signed 12-bit immediate.  Encoded: first word = the partner's low 20 bits
 *     above an AUIPC opcode with rd = x2 (so rs1, i.e. the old rd, lands in bits 31:27); second word = the absolute target, big endian.
 *     Next: i + 8.  Without such a partner: i + 6.
 *   AUIPC x0 / x2: an encoded pair looks exactly like "AUIPC x2" with bits 13:12 = 11 and bits 31:27 not x0 / x2.  A real instruction
 *     of that shape is escaped by exchanging fields with the next word (first = AUIPC with rd = its old bits 31:27 and the next word's
 *     upper 20 bits; second = its old bits 31:12 below the next word's low 12 bits), and decoding reverses that.  Next: i + 8.  An
 *     AUIPC x0 / x2 of any other shape: i + 4.
 *   anything else: i + 2.
 * The decoder makes the same decisions on the encoded bytes: it sees an encoded pair as the AUIPC x2 shape above and an escaped one
 * as an AUIPC with a partner. */
#include <stddef.h>
#include <stdint.h>

static uint32_t ld_le(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static uint32_t ld_be(const uint8_t *p) { return (uint32_t)p[3] | ((uint32_t)p[2] << 8) | ((uint32_t)p[1] << 16) | ((uint32_t)p[0] << 24); }
static void st_le(uint8_t *p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }
static void st_be(uint8_t *p, uint32_t v) { p[3] = (uint8_t)v; p[2] = (uint8_t)(v >> 8); p[1] = (uint8_t)(v >> 16); p[0] = (uint8_t)(v >> 24); }

/* in place on d[0 .. n); pc = the start offset (the address of d[0]); enc: 1 encode, 0 decode */
void b2zo_riscv(int enc, uint8_t *d, size_t n, uint32_t pc) {
    const size_t end = n & ~(size_t)1;
    for (size_t i = 0; i + 8 <= end;) {
        const uint32_t w = ld_le(d + i), op = w & 0x7F, rd = (w >> 7) & 0x1F, at = pc + (uint32_t)i;
        if (op == 0x6F) {                                           /* JAL */
            if (rd != 1 && rd != 5) { i += 2; continue; }
            if (enc) {
                const uint32_t off = (((w >> 31) & 1) << 20) | (((w >> 21) & 0x3FF) << 1) | (((w >> 20) & 1) << 11) | (((w >> 12) & 0xFF) << 12);
                const uint32_t t = off + at;
                d[i + 1] = (uint8_t)((d[i + 1] & 0x0F) | (((t >> 17) & 0xF) << 4));
                d[i + 2] = (uint8_t)(t >> 9); d[i + 3] = (uint8_t)(t >> 1);
            } else {
                const uint32_t t = ((uint32_t)(d[i + 1] >> 4) << 17) | ((uint32_t)d[i + 2] << 9) | ((uint32_t)d[i + 3] << 1);
                const uint32_t off = t - at;
                st_le(d + i, (w & 0xFFF) | (((off >> 20) & 1) << 31) | (((off >> 1) & 0x3FF) << 21) | (((off >> 11) & 1) << 20) | (((off >> 12) & 0xFF) << 12));
            }
            i += 4;
        } else if (op == 0x17) {                                    /* AUIPC */
            const uint32_t x = ld_le(d + i + 4);
            if (rd != 0 && rd != 2) {
                if ((x & 3) != 3 || ((x >> 15) & 0x1F) != rd) { i += 6; continue; }
                if (enc) {
                    const int32_t lo12 = (int32_t)x >> 20;
                    st_le(d + i, (x << 12) | (2u << 7) | 0x17);
                    st_be(d + i + 4, (w & 0xFFFFF000u) + (uint32_t)lo12 + at);
                } else {                                            /* an escaped AUIPC x2 */
                    st_le(d + i, (x << 12) | (2u << 7) | 0x17);
                    st_le(d + i + 4, (w & 0xFFFFF000u) | (x >> 20));
                }
                i += 8;
            } else {
                const uint32_t hi5 = w >> 27;
                if (rd != 2 || ((w >> 12) & 3) != 3 || hi5 == 0 || hi5 == 2) { i += 4; continue; }
                if (enc) {                                          /* escape a real AUIPC x2 of the encoded shape */
                    st_le(d + i, (hi5 << 7) | 0x17 | (x & 0xFFFFF000u));
                    st_le(d + i + 4, (w >> 12) | (x << 20));
                } else {                                            /* an encoded pair: rebuild AUIPC rd + partner */
                    const uint32_t t = ld_be(d + i + 4) - at;       /* target - address = (upper << 12) + sign-extended lo12 */
                    const uint32_t upper = (t + 0x800) & 0xFFFFF000u;
                    st_le(d + i, (hi5 << 7) | 0x17 | upper);
                    st_le(d + i + 4, (w >> 12) | (t << 20));
                }
                i += 8;
            }
        } else i += 2;
    }
}
